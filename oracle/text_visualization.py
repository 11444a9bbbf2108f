"""Word-importance oracle of the BERT notebook (TEST INFRASTRUCTURE, host, numpy).

``BERT_explainability.ipynb`` explains a sentence with ``generate_LRP(start_layer=0)`` and then, on the [S] map ``expl``:

    expl = (expl - expl.min()) / (expl.max() - expl.min())          # fp32 torch ops, one rounding each
    if class_name == "NEGATIVE": expl *= (-1)

before handing it to captum's ``visualization.visualize_text``.  Restated here over the first L tokens of a padded row,
with the engine's conventions where the notebook has none: a constant row gives 0 (the notebook's 0 / 0 would be NaN),
NaN anywhere in the row makes the row NaN (``torch.min`` / ``torch.max`` propagate it), and the padding is 0.

Captum (not installed here) is restated for the parts the command reproduces, ``captum/attr/_utils/visualization.py``
(0.6.0): ``_get_color`` (the score clipped to [-1, 1] in double precision; hsl(120, 75%, 100 - int(50 a)%) above 0,
hsl(0, 75%, 100 - int(-40 a)%) otherwise), ``format_classname``, ``format_special_tokens``, ``format_word_importances`` and
the table and legend of ``visualize_text``.  Text is HTML-escaped (captum writes it raw).
"""
import html

import numpy as np


def normalize(row, length, sign):
    """fp32 [S] -> fp32 [S]: ((a - min) / (max - min)) * sign over a = row[:length], 0 for a constant row, zeros after."""
    a = np.asarray(row, dtype=np.float32)[:length]
    out = np.zeros(np.asarray(row).shape[0], dtype=np.float32)
    if np.isnan(a).any():
        out[:length] = np.float32(np.nan)
        return out
    mn, mx = a.min(), a.max()
    if mx == mn:
        return out
    with np.errstate(invalid="ignore"):
        out[:length] = ((a - mn) / (mx - mn)) * np.float32(sign)
    return out


def sign_of(class_name):
    """The notebook flips the map of a class named NEGATIVE ("higher explanation scores are more negative")."""
    return -1.0 if class_name == "NEGATIVE" else 1.0


def color(a):
    a = float(a)
    a = max(-1, min(1, a))
    if a > 0:
        return "hsl(%d, %d%%, %d%%)" % (120, 75, 100 - int(50 * a))
    return "hsl(%d, %d%%, %d%%)" % (0, 75, 100 - int(-40 * a))


def classname_cell(name):
    return '<td><text style="padding-right:2em"><b>' + html.escape(str(name)) + "</b></text></td>"


def special_token(tok):
    return "#" + tok.strip("<>") if tok.startswith("<") and tok.endswith(">") else tok


def mark(tok, a):
    return ('<mark style="background-color: ' + color(a) + '; opacity:1.0; line-height:1.75"><font color="black"> '
            + html.escape(special_token(tok)) + " </font></mark>")


def table(records):
    """The page: legend, header row, one row per record (true label = attribution label = the explained class)."""
    legend = "".join('<span style="display: inline-block; width: 10px; height: 10px; border: 1px solid; '
                     'background-color: ' + color(v) + '"></span> ' + lab + "  "
                     for v, lab in ((-1, "Negative"), (0, "Neutral"), (1, "Positive")))
    rows = ""
    for r in records:
        rows += ("<tr>" + classname_cell(r["explained_label"])
                 + classname_cell("%s (%.2f)" % (r["predicted_label"], r["predicted_probability"]))
                 + classname_cell(r["explained_label"]) + classname_cell("%.2f" % sum(r["scores"]))
                 + "<td>" + "".join(mark(t, a) for t, a in zip(r["tokens"], r["scores"])) + "</td>" + "<tr>")
    return ('<table width: 100%><div style="border-top: 1px solid; margin-top: 5px; padding-top: 5px; '
            'display: inline-block"><b>Legend: </b>' + legend + "</div>"
            "<tr><th>True Label</th><th>Predicted Label</th><th>Attribution Label</th><th>Attribution Score</th>"
            "<th>Word Importance</th>" + rows + "</table>")


def records(tokens, token_types, scores, probs, names, explained=None):
    """The JSON records of a batch from host arrays: tokens / token_types per row (unpadded), scores fp32 [B, S], probs
    fp32 [B, C]; explained [B] (default: the arg-max of probs)."""
    out = []
    probs = np.asarray(probs, dtype=np.float32)
    for b in range(len(tokens)):
        p = int(np.argmax(probs[b]))
        e = p if explained is None else int(explained[b])
        n = len(tokens[b])
        out.append({"tokens": list(tokens[b]), "token_type_ids": [int(v) for v in token_types[b]],
                    "scores": [float(v) for v in np.asarray(scores[b], dtype=np.float32)[:n]],
                    "predicted_class": p, "predicted_label": names[p], "predicted_probability": float(probs[b, p]),
                    "explained_class": e, "explained_label": names[e], "explained_probability": float(probs[b, e])})
    return out
