"""Segmentation-evaluation oracle (TEST INFRASTRUCTURE, CPU torch / numpy).

Restates ``/root/reference/baselines/ViT/imagenet_seg_eval.py`` from the explanation map on:

* ``normalised_map``    ``:212-217``: bilinear x16 (``F.interpolate``; not for ``full_lrp``), then ``(Res - min) / (max - min)``
* ``sample_metrics``    ``:219-275``: threshold at ``Res.mean()``, the arg-max of ``cat(Res_0, Res_1)`` (pixel accuracy,
                        intersection / union of ``utils/metrices.py:135-177``), F1 on ``Res_1``, AP of ``cat(1 - Res, Res)``
                        against the one-hot label, and the PR-curve scores ``Res.clamp(min=thr) / Res.max()`` — the
                        reference's torch ops, literally, including the in-place NaN zeroing through the ``Res_1_AP`` alias
* ``totals``            ``:280-309``: pixAcc, IoU, mIoU, mAP, mF1 with the ``np.spacing(1)`` formulas
* ``binary_clf_curve`` / ``precision_recall_curve`` / ``average_precision`` / ``f1``: numpy restatements of sklearn 1.x
  (``_binary_clf_curve`` with ties grouped by equal score, ``precision_recall_curve`` without ``drop_intermediate``,
  ``average_precision_score`` as the step integral clipped at 0, ``f1_score`` with zero division -> 0), so that the GPU
  machine does not need sklearn.
"""
import numpy as np
import torch
import torch.nn.functional as F


def binary_clf_curve(y_true, y_score):
    """(fps, tps, thresholds) per distinct score, descending; tps / fps float64 like sklearn's."""
    y_true = np.asarray(y_true).reshape(-1)
    y_score = np.asarray(y_score).reshape(-1)
    order = np.argsort(y_score, kind="stable")[::-1]
    y_score = y_score[order]
    y_true = (y_true[order] == 1).astype(np.float64)
    distinct = np.nonzero(np.diff(y_score))[0]
    idx = np.concatenate([distinct, [y_true.size - 1]])
    tps = np.cumsum(y_true, dtype=np.float64)[idx]
    fps = 1 + idx.astype(np.float64) - tps
    return fps, tps, y_score[idx]


def pr_from_counts(tps, fps):
    """sklearn 1.x ``precision_recall_curve`` from the curve counts: reversed, with 1 / 0 appended, no truncation."""
    tps = np.asarray(tps, dtype=np.float64)
    fps = np.asarray(fps, dtype=np.float64)
    ps = tps + fps
    with np.errstate(invalid="ignore", divide="ignore"):
        precision = np.where(ps != 0, tps / ps, 0.0)
    recall = np.ones_like(tps) if tps[-1] == 0 else tps / tps[-1]
    return np.hstack((precision[::-1], 1.0)), np.hstack((recall[::-1], 0.0))


def precision_recall_curve(y_true, y_score):
    fps, tps, thr = binary_clf_curve(y_true, y_score)
    precision, recall = pr_from_counts(tps, fps)
    return precision, recall, thr[::-1]


def average_precision(y_true, y_score):
    precision, recall, _ = precision_recall_curve(y_true, y_score)
    return float(max(0.0, -np.sum(np.diff(recall) * precision[:-1])))


def f1(tp, fp, fn):
    """``f1_score`` of a binary mask: 2 TP / (2 TP + FP + FN) in float64, 0 when the denominator is 0."""
    denom = 2 * tp + fp + fn
    return float(2 * tp) / float(denom) if denom else 0.0


def normalised_map(raw, scale=16):
    """raw map (g*g values) -> Res [1,1,G,G] fp32, min-max normalised (``:212-217``)."""
    g = int(round(raw.numel() ** 0.5))
    Res = raw.reshape(1, 1, g, g).to(torch.float32)
    if scale != 1:
        Res = torch.nn.functional.interpolate(Res, scale_factor=scale, mode='bilinear')
    return (Res - Res.min()) / (Res.max() - Res.min())


def sample_metrics(raw, label, scale=16, thr=0., threshold=None):
    """``eval_batch`` (``:217-275``) of one sample from its raw map.  ``threshold`` overrides ``Res.mean()`` (to compare
    counts at another implementation's threshold).  Returns a dict: mean (np.float32), tp / fp / fn / tn, correct,
    labeled, inter [2], union [2], ap (float64), f1 (float64 [G], one per image row), pred (fp32 [P]), target (int64 [P])."""
    Res = normalised_map(raw, scale)
    G = Res.shape[-1]
    ret = Res.mean()
    t = ret if threshold is None else torch.tensor(threshold, dtype=torch.float32)
    Res_1 = Res.gt(t).type(Res.type())
    Res_0 = Res.le(t).type(Res.type())
    Res_1_AP = Res
    Res_0_AP = 1 - Res
    Res_1[Res_1 != Res_1] = 0
    Res_0[Res_0 != Res_0] = 0
    Res_1_AP[Res_1_AP != Res_1_AP] = 0               # in place on Res
    Res_0_AP[Res_0_AP != Res_0_AP] = 0
    pred = (Res.clamp(min=thr) / Res.max()).reshape(-1).numpy()
    output = torch.cat((Res_0, Res_1), 1)
    output_AP = torch.cat((Res_0_AP, Res_1_AP), 1)
    lab = torch.as_tensor(label).reshape(G, G).long()
    _, predict = torch.max(output[0], 0)
    fg, pos = predict == 1, lab == 1
    tp, fp = int((fg & pos).sum()), int((fg & ~pos).sum())
    fn, tn = int((~fg & pos).sum()), int((~fg & ~pos).sum())
    # get_f1_scores(output[0, 1], labels[0]) (metrices.py:26-38) takes the first dimension of its input as the batch: one F1
    # per image row
    f1_rows = np.array([f1(int((fg[r] & pos[r]).sum()), int((fg[r] & ~pos[r]).sum()), int((~fg[r] & pos[r]).sum()))
                        for r in range(G)])
    onehot = torch.cat([(lab == 0), (lab == 1)]).reshape(-1).long().numpy()
    ap = float(np.nan_to_num(average_precision(onehot, output_AP[0].reshape(-1).numpy())))
    return {"mean": np.float32(ret.item()), "tp": tp, "fp": fp, "fn": fn, "tn": tn, "correct": tp + tn, "labeled": G * G,
            "inter": np.array([tn, tp], dtype=np.int64), "union": np.array([tn + fp + fn, tp + fp + fn], dtype=np.int64),
            "ap": ap, "f1": f1_rows, "pred": pred, "target": lab.reshape(-1).numpy()}


def totals(correct, labeled, inter, union, ap, f1s):
    """``:299-309`` after the last sample: (pixAcc, IoU [2], mIoU, mAP, mF1).  ap / f1s are per-sample lists (the
    reference keeps one-element AP arrays and [G] row-F1 arrays; the means run over the same values in the same order)."""
    total_correct = np.int64(np.sum(np.asarray(correct, dtype=np.int64)))
    total_label = np.int64(np.sum(np.asarray(labeled, dtype=np.int64)))
    total_inter = np.asarray(inter, dtype=np.int64).reshape(-1, 2).sum(0)
    total_union = np.asarray(union, dtype=np.int64).reshape(-1, 2).sum(0)
    pixAcc = np.float64(1.0) * total_correct / (np.spacing(1, dtype=np.float64) + total_label)
    IoU = np.float64(1.0) * total_inter / (np.spacing(1, dtype=np.float64) + total_union)
    mIoU = IoU.mean()
    mAp = np.mean([np.array([a]) for a in ap])
    mF1 = np.mean([np.asarray(f) for f in f1s])
    return {"pixAcc": float(pixAcc), "IoU": IoU, "mIoU": float(mIoU), "mAP": float(mAp), "mF1": float(mF1)}


def evaluate(raw_maps, labels, scale=16, thr=0.):
    """Every sample, the totals and the PR curve over all pixels (``:312-314``)."""
    per = [sample_metrics(m, l, scale=scale, thr=thr) for m, l in zip(raw_maps, labels)]
    tot = totals([p["correct"] for p in per], [p["labeled"] for p in per], [p["inter"] for p in per],
                 [p["union"] for p in per], [p["ap"] for p in per], [p["f1"] for p in per])
    precision, recall, _ = precision_recall_curve(np.concatenate([p["target"] for p in per]),
                                                  np.concatenate([p["pred"] for p in per]))
    return per, tot, precision, recall


def pr_summary(precision, recall, points=64):
    """What the fixture stores of a PR curve: length, sums, ``points`` strided samples and the first / last 16 values."""
    out = {}
    for name, a in (("precision", np.asarray(precision)), ("recall", np.asarray(recall))):
        idx = np.linspace(0, len(a) - 1, points).astype(np.int64)
        out[name + "_len"] = np.int64(len(a))
        out[name + "_sum"] = np.float64(np.sum(a))
        out[name + "_strided"] = a[idx]
        out[name + "_head"] = a[:16]
        out[name + "_tail"] = a[-16:]
    return out
