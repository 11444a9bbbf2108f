"""The word-importance view of the BERT notebook (``BERT_explainability.ipynb``) as a command, for sentences and sentence
pairs.

    python -m transformer_explainability_b200.text_visualization --model-dir bert-base-uncased-SST-2/ \\
        --text "This movie was the best movie I have ever seen!" --labels NEGATIVE POSITIVE --output-dir out/

    python -m transformer_explainability_b200.text_visualization --model-dir mnli/ --text "A man plays." \\
        --text-pair "Somebody is playing." --output-dir out/

``--model-dir`` is a local Hugging Face directory (``config.json``, the tokenizer's files, ``model.safetensors`` or
``pytorch_model.bin``), the layout ``from_pretrained`` leaves on disk; nothing is downloaded.  ``config.json``'s
``model_type`` picks the classifier: ``bert``, ``roberta``, ``xlm-roberta`` or ``distilbert`` (``MODEL_TYPES``).  The notebook explains a
sentence with ``generate_LRP(start_layer=0)``, min-max normalises the map, negates it when the explained class is named
``NEGATIVE``, and shows captum's ``visualize_text`` table with the probability of the class.  Here, per batch of
``--batch-size`` sentences, tokenised as the notebook tokenises them (a pair with its ``token_type_ids``) and padded to the
batch's longest, the library launches F + A + 2 kernels (``te_kernel_launch_count``): the F launches of one engine forward
and the A of its ``attribute`` (one ``explain`` call), one ``te_class_probs`` and one ``te_token_importance``; then one
device-to-host copy carries the scores, the probabilities and the classes.  Two files are written:

``word_importance.json``  per sentence its text (and pair), tokens, segment ids, scores, the predicted class and the
                          explained class with their names and probabilities;
``word_importance.html``  captum ``visualize_text``'s table (true label, predicted label (prob), attribution label,
                          attribution score, word importance) with its legend.  The command has no true labels: that
                          column holds the explained class, as the notebook's records do.

The colour of each word is captum's ``_get_color`` on the host, in double precision from the fp32 score, so that
``int(50 * a)`` rounds as captum's Python does (the device's fp32 product can land on the other side of an integer).
"""
import argparse
import html
import json
import os

import numpy as np
import torch

from ._host import to_host
from .visualization import METHODS, _check_method


# ---- host formatting (captum.attr.visualization's visualize_text layout) --------------------------------------------------
def get_color(attr):
    """captum's ``_get_color``: the score clipped to [-1, 1]; green ``hsl(120, 75%, L%)`` with L = 100 - int(50 a) for
    a > 0, else red ``hsl(0, 75%, L%)`` with L = 100 - int(-40 a).  ``attr`` is taken in double precision."""
    attr = max(-1, min(1, float(attr)))
    if attr > 0:
        return "hsl(120, 75%, {}%)".format(100 - int(50 * attr))
    return "hsl(0, 75%, {}%)".format(100 - int(-40 * attr))


def _cell(text):
    return '<td><text style="padding-right:2em"><b>{}</b></text></td>'.format(html.escape(str(text)))


def _word(token):
    if token.startswith("<") and token.endswith(">"):
        token = "#" + token.strip("<>")
    return html.escape(token)


def word_importances_html(tokens, scores):
    tags = ["<td>"]
    for tok, a in zip(tokens, scores):
        tags.append('<mark style="background-color: {}; opacity:1.0; line-height:1.75"><font color="black"> {} </font>'
                    '</mark>'.format(get_color(a), _word(tok)))
    tags.append("</td>")
    return "".join(tags)


def render_html(records):
    """captum ``visualize_text``'s table and legend for ``records`` (dicts as written to ``word_importance.json``)."""
    dom = ["<table width: 100%>",
           '<div style="border-top: 1px solid; margin-top: 5px; padding-top: 5px; display: inline-block">',
           "<b>Legend: </b>"]
    for value, label in zip((-1, 0, 1), ("Negative", "Neutral", "Positive")):
        dom.append('<span style="display: inline-block; width: 10px; height: 10px; border: 1px solid; '
                   'background-color: {}"></span> {}  '.format(get_color(value), label))
    dom.append("</div>")
    dom.append("<tr><th>True Label</th><th>Predicted Label</th><th>Attribution Label</th><th>Attribution Score</th>"
               "<th>Word Importance</th>")
    for r in records:
        dom.append("".join(["<tr>", _cell(r["explained_label"]),
                            _cell("{0} ({1:.2f})".format(r["predicted_label"], r["predicted_probability"])),
                            _cell(r["explained_label"]), _cell("{0:.2f}".format(sum(r["scores"]))),
                            word_importances_html(r["tokens"], r["scores"]), "<tr>"]))
    dom.append("</table>")
    return "".join(dom)


# ---- model and tokenizer -------------------------------------------------------------------------------------------------
# config.json model_type -> (transformers config class, the engine's classifier: module, class)
_M = "transformer_explainability_b200.BERT_explainability.modules.BERT."
MODEL_TYPES = {
    "bert": ("BertConfig", _M + "BertForSequenceClassification", "BertForSequenceClassification"),
    "roberta": ("RobertaConfig", _M + "RobertaForSequenceClassification", "RobertaForSequenceClassification"),
    "xlm-roberta": ("XLMRobertaConfig", _M + "RobertaForSequenceClassification", "XLMRobertaForSequenceClassification"),
    "distilbert": ("DistilBertConfig", _M + "DistilBertForSequenceClassification",
                   "DistilBertForSequenceClassification"),
}


def load_model(model_dir, device="cuda"):
    """The engine's classifier for ``config.json``'s ``model_type`` (``MODEL_TYPES``) with the weights of a local Hugging
    Face directory."""
    import importlib
    import transformers
    with open(os.path.join(model_dir, "config.json")) as f:
        model_type = json.load(f).get("model_type", "bert")
    if model_type not in MODEL_TYPES:
        raise ValueError("%s: model_type %r is not supported; the supported types are %s"
                         % (model_dir, model_type, ", ".join(sorted(MODEL_TYPES))))
    config_cls, module, cls = MODEL_TYPES[model_type]
    config = getattr(transformers, config_cls).from_json_file(os.path.join(model_dir, "config.json"))
    st = os.path.join(model_dir, "model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file
        sd = load_file(st)
    else:
        sd = torch.load(os.path.join(model_dir, "pytorch_model.bin"), map_location="cpu", weights_only=True)
    model = getattr(importlib.import_module(module), cls)(config)
    res = model.load_state_dict(sd, strict=False)
    missing = [k for k in res.missing_keys if "position_ids" not in k]
    if missing:
        raise KeyError("%s lacks %s" % (model_dir, ", ".join(missing[:5])))
    return model.to(device).eval()


def load_tokenizer(model_dir):
    from transformers import AutoTokenizer
    return AutoTokenizer.from_pretrained(model_dir, local_files_only=True)


def tokenize(tokenizer, texts, pairs=None, max_length=512):
    """The notebook's ``tokenizer(text_batch, return_tensors='pt')``, with the second sentence of each pair and padding
    to the longest: (input_ids, token_type_ids, attention_mask) int64 [B, S] on the host."""
    enc = tokenizer(list(texts), list(pairs) if pairs is not None else None, padding=True, truncation=True,
                    max_length=max_length, return_tensors="pt", return_token_type_ids=True, return_attention_mask=True)
    return enc["input_ids"], enc["token_type_ids"], enc["attention_mask"]


def class_names(config, labels=None):
    n = config.num_labels
    if labels:
        if len(labels) != n:
            raise ValueError("--labels needs %d names, got %d" % (n, len(labels)))
        return list(labels)
    id2label = getattr(config, "id2label", None) or {}
    return [str(id2label.get(i, id2label.get(str(i), "LABEL_%d" % i))) for i in range(n)]


# ---- one batch on the device ---------------------------------------------------------------------------------------------
def explain_batch(model, ids, tt, mask, names, class_index=None, start_layer=0, method="transformer_attribution"):
    """One batch on the device: one engine ``explain`` (``return_logits``), ``te_class_probs``, ``te_token_importance``,
    one device-to-host copy.  Returns host arrays (scores fp32 [B, S] with zeros past each length, probs fp32 [B, C],
    explained int64 [B], predicted int64 [B])."""
    from . import _lib, ops
    _check_method(method)
    eng = model.engine()
    dev = eng.device
    flags = eng.flags | (_lib.FLAG_ATTN_GRAD_ROLLOUT if method == "attn_grad_rollout" else 0)
    # segment ids reach the engine only for a model with a token-type table (DistilBERT has none)
    tt_dev = tt.to(dev) if eng.cfg.type_vocab > 0 else None
    maps, idx, logits = eng.explain(ids.to(dev), mask.to(dev), index=class_index, start_layer=start_layer, flags=flags,
                                    return_logits=True, token_type_ids=tt_dev)
    lengths = mask.sum(dim=1).to(torch.int32)
    neg = torch.tensor([-1.0 if n == "NEGATIVE" else 1.0 for n in names], dtype=torch.float32, device=dev)
    sign = neg[idx.long()]
    scores, probs, explained = to_host(ops.token_importance(maps, lengths.to(dev), sign), ops.class_probs(logits), idx)
    return scores, probs, explained.astype(np.int64), probs.argmax(axis=1).astype(np.int64)


def records_for(tokenizer, texts, pairs, ids, tt, mask, scores, probs, explained, predicted, names):
    out = []
    for b in range(len(texts)):
        n = int(mask[b].sum())
        e, p = int(explained[b]), int(predicted[b])
        out.append({"text": texts[b], "text_pair": pairs[b] if pairs is not None else None,
                    "tokens": tokenizer.convert_ids_to_tokens(ids[b, :n].tolist()),
                    "token_type_ids": [int(v) for v in tt[b, :n]],
                    "scores": [float(v) for v in scores[b, :n]],
                    "predicted_class": p, "predicted_label": names[p], "predicted_probability": float(probs[b, p]),
                    "explained_class": e, "explained_label": names[e], "explained_probability": float(probs[b, e])})
    return out


def write_outputs(records, output_dir):
    os.makedirs(output_dir, exist_ok=True)
    paths = os.path.join(output_dir, "word_importance.json"), os.path.join(output_dir, "word_importance.html")
    with open(paths[0], "w") as f:
        json.dump(records, f, indent=1)
    with open(paths[1], "w") as f:
        f.write(render_html(records))
    return paths


def run(model, tokenizer, texts, pairs=None, names=None, class_index=None, start_layer=0,
        method="transformer_attribution", batch_size=16, output_dir="."):
    """The command on already-parsed arguments; returns (records, written paths)."""
    names = names or class_names(model.config)
    records = []
    for s in range(0, len(texts), batch_size):
        tx = texts[s:s + batch_size]
        px = pairs[s:s + batch_size] if pairs is not None else None
        ids, tt, mask = tokenize(tokenizer, tx, px, model.max_length())
        scores, probs, explained, predicted = explain_batch(model, ids, tt, mask, names, class_index, start_layer, method)
        records += records_for(tokenizer, tx, px, ids, tt, mask, scores, probs, explained, predicted, names)
    return records, write_outputs(records, output_dir)


def build_parser():
    p = argparse.ArgumentParser(description="The BERT notebook's word-importance view for sentences and sentence pairs, "
                                            "for BERT, RoBERTa, XLM-RoBERTa and DistilBERT classifiers")
    p.add_argument("--model-dir", required=True,
                   help="local Hugging Face directory: config.json (model_type %s), the tokenizer's files, "
                        "model.safetensors or pytorch_model.bin" % " / ".join(MODEL_TYPES))
    p.add_argument("--text", action="append", required=True, help="a sentence (repeat for more)")
    p.add_argument("--text-pair", action="append", default=None,
                   help="the second sentence of the pair, one per --text (repeat in the same order)")
    p.add_argument("--class-index", type=int, default=None, help="the class explained (default: the predicted one)")
    p.add_argument("--labels", nargs="+", default=None, help="class names, overriding config.id2label")
    p.add_argument("--start-layer", type=int, default=0)
    p.add_argument("--method", choices=METHODS, default="transformer_attribution")
    p.add_argument("--batch-size", type=int, default=16)
    p.add_argument("--output-dir", required=True)
    return p


def parse_args(argv=None):
    p = build_parser()
    args = p.parse_args(argv)
    if args.batch_size < 1:
        p.error("--batch-size must be at least 1")
    if args.text_pair is not None and len(args.text_pair) != len(args.text):
        p.error("--text-pair must be given once per --text (%d, got %d)" % (len(args.text), len(args.text_pair)))
    if args.start_layer < 0:
        p.error("--start-layer must be non-negative")
    return args


def main(argv=None):
    args = parse_args(argv)
    model = load_model(args.model_dir)
    names = class_names(model.config, args.labels)
    if args.class_index is not None and not 0 <= args.class_index < len(names):
        raise SystemExit("--class-index must lie in 0..%d" % (len(names) - 1))
    if args.start_layer >= model.config.num_hidden_layers:
        raise SystemExit("--start-layer must lie in 0..%d" % (model.config.num_hidden_layers - 1))
    records, paths = run(model, load_tokenizer(args.model_dir), args.text, args.text_pair, names, args.class_index,
                         args.start_layer, args.method, args.batch_size, args.output_dir)
    print("%d sentences: %s" % (len(records), " ".join(paths)))
    return paths


if __name__ == "__main__":
    main()
