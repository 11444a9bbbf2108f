"""ImageNet-segmentation evaluation of the ViT explanation methods (``baselines/ViT/imagenet_seg_eval.py``).

Each method's map is up-sampled to the image (bilinear x16; ``full_lrp`` is already per pixel), min-max normalised and
thresholded at its mean; the evaluation reports pixel accuracy, the IoU of background / foreground and their mean, the mean
average precision and the mean F1 over the images, and the precision-recall curve over every pixel of the set — Table 1
of the paper.  Per data batch: one batched engine call makes the maps, one ``te_seg_metrics`` call computes every
per-sample metric (counts, AP over sorted keys) and emits the PR-curve keys, which stay on the device, and one small
device-to-host copy brings back the counts and AP.  At the end the PR keys are sorted once (``te_sort_keys_u32``) and
reduced to the curve (``te_pr_curve``).

    python -m transformer_explainability_b200.segmentation --method transformer_attribution \\
        --imagenet-seg-path gtsegs_ijcv.mat --state-dict vit_base_patch16_224.pth

Deviations from the reference script (DESIGN.md §1):
 * batches larger than 1: every min / max / mean is taken per sample, which is what the reference computes at its
   hard-coded batch size 1; the results do not depend on the batch size;
 * the mean threshold is accumulated in fp64 and rounded once to fp32; torch's ``Res.mean()`` may differ by 1 ulp, which
   only moves pixels exactly at the mean;
 * a degenerate map (constant, max == min) enters the PR curve with score 0 and is counted in ``degenerate``; the
   reference's score is NaN there and its final ``precision_recall_curve`` raises;
 * ``--is-ablation`` parses a real boolean (the reference's ``type=bool`` turns ``--is-ablation False`` into True);
 * ``--method lrp`` is rejected (the reference lists it but fails with a ``NameError``), and so is ``--save-img``.
"""
import argparse
import glob
import os

import numpy as np
import torch

from . import ops
from .perturbation import str2bool

METHODS = ("rollout", "transformer_attribution", "full_lrp", "lrp_last_layer", "attn_last_layer", "attn_gradcam")
_MODEL = {"rollout": "new", "attn_gradcam": "new", "transformer_attribution": "lrp", "full_lrp": "orig",
          "lrp_last_layer": "orig", "attn_last_layer": "orig"}


# ---- data ----------------------------------------------------------------------------------------------------------------
def seg_transforms():
    """(image transform, label transform) of the reference (``:122-130``): Resize 224 + ToTensor + Normalize(0.5, 0.5), and
    Resize 224 NEAREST."""
    import torchvision.transforms as transforms
    from PIL import Image
    normalize = transforms.Normalize(mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5])
    img = transforms.Compose([transforms.Resize((224, 224)), transforms.ToTensor(), normalize])
    lbl = transforms.Compose([transforms.Resize((224, 224), Image.NEAREST)])
    return img, lbl


class ImagenetSegmentation(torch.utils.data.Dataset):
    """``Imagenet_Segmentation`` of ``data/Imagenet.py:42-81``: image / mask pairs of ``gtsegs_ijcv.mat`` (MATLAB v7.3,
    read through h5py's object references).  ``[i]`` -> (image, label int64 [224,224]) with the given transforms."""

    def __init__(self, path, transform=None, target_transform=None):
        try:
            import h5py
        except ImportError as e:
            raise ImportError("ImagenetSegmentation reads %s (MATLAB v7.3, HDF5 object references) through h5py; "
                              "install h5py" % path) from e
        self.path = path
        self.transform = transform
        self.target_transform = target_transform
        self.h5py = None
        with h5py.File(path, "r") as f:
            self.data_length = len(f["/value/img"])

    def __len__(self):
        return self.data_length

    def __getitem__(self, index):
        import h5py
        from PIL import Image
        if self.h5py is None:
            self.h5py = h5py.File(self.path, "r")
        f = self.h5py
        img = np.array(f[f["/value/img"][index, 0]]).transpose((2, 1, 0))
        target = np.array(f[f[f["/value/gt"][index, 0]][0, 0]]).transpose((1, 0))
        img = Image.fromarray(img).convert("RGB")
        target = Image.fromarray(target)
        if self.transform is not None:
            img = self.transform(img)
        if self.target_transform is not None:
            target = torch.from_numpy(np.array(self.target_transform(target)).astype("int32")).long()
        return img, target

    def __getstate__(self):                      # DataLoader workers open the file themselves
        state = dict(self.__dict__)
        state["h5py"] = None
        return state


# ---- the evaluation ------------------------------------------------------------------------------------------------------
def check_method(method):
    if method not in METHODS:
        raise ValueError("unknown segmentation method %r (expected one of %s)" % (method, ", ".join(METHODS)))


def explain(method, x, lrp=None, orig_lrp=None, baselines=None, is_ablation=False):
    """The map of ``method`` for x [B,3,H,W] as the reference makes it (``:187-210``), batched -> [B, values]."""
    check_method(method)
    gen = {"new": baselines, "lrp": lrp, "orig": orig_lrp}[_MODEL[method]]
    if gen is None:
        raise ValueError("method %r needs the %s generator" % (method, {"new": "baselines", "lrp": "lrp",
                                                                         "orig": "orig_lrp"}[_MODEL[method]]))
    if method == "rollout":
        res = gen.generate_rollout(x, start_layer=1)
    elif method == "transformer_attribution":
        res = gen.generate_LRP_batched(x, start_layer=1)
    elif method == "full_lrp":
        res = gen.generate_LRP(x, method="full")
    elif method == "lrp_last_layer":
        res = gen.generate_LRP(x, method="last_layer", is_ablation=is_ablation)
    elif method == "attn_last_layer":
        res = gen.generate_LRP(x, method="last_layer_attn", is_ablation=is_ablation)
    else:
        res = gen.generate_cam_attn(x)
    return res.reshape(x.shape[0], -1).to(torch.float32).contiguous()


def totals(correct, labeled, inter, union, ap, f1):
    """The reference's running totals after the last sample (``:299-309``)."""
    eps = np.spacing(1, dtype=np.float64)
    pixAcc = np.float64(1.0) * np.int64(np.sum(correct)) / (eps + np.int64(np.sum(labeled)))
    IoU = np.float64(1.0) * np.asarray(inter, dtype=np.int64).reshape(-1, 2).sum(0) / \
        (eps + np.asarray(union, dtype=np.int64).reshape(-1, 2).sum(0))
    return {"pixAcc": float(pixAcc), "IoU": IoU, "mIoU": float(IoU.mean()),
            "mAP": float(np.mean(np.asarray(ap, dtype=np.float64).reshape(-1, 1))),
            "mF1": float(np.mean(np.asarray(f1, dtype=np.float64)))}


def precision_recall(tps, fps):
    """sklearn 1.x ``precision_recall_curve`` from the curve counts (descending thresholds): precision = tps / (tps + fps),
    recall = tps / tps[-1], both reversed, with 1 / 0 appended; no full-recall truncation."""
    tps = np.asarray(tps, dtype=np.float64)
    fps = np.asarray(fps, dtype=np.float64)
    if tps.size == 0:
        return np.ones(1), np.zeros(1)
    ps = tps + fps
    with np.errstate(invalid="ignore", divide="ignore"):
        precision = np.where(ps != 0, tps / ps, 0.0)
    recall = np.ones_like(tps) if tps[-1] == 0 else tps / tps[-1]
    return np.hstack((precision[::-1], 1.0)), np.hstack((recall[::-1], 0.0))


def segmentation_eval(method, loader, lrp=None, orig_lrp=None, baselines=None, thr=0., is_ablation=False, pr_curve=True):
    """The loop of ``imagenet_seg_eval.py`` (``:170-314``) on the engine.  ``loader`` yields (images [B,3,224,224]
    normalised, labels [B,224,224] of 0 / 1); ``lrp`` / ``orig_lrp`` / ``baselines`` are this package's generators over
    ``ViT_LRP`` / ``ViT_orig_LRP`` / ``ViT_new`` models (only the one ``method`` uses is needed).
    Returns a dict: per sample ``correct, labeled`` [N], ``inter, union`` [N,2] (background, foreground), ``ap`` [N] and
    ``f1`` [N, 224] float64 (the reference's F1 is taken per image row: ``get_f1_scores`` treats the first dimension of the
    mask as its batch), ``mean`` [N] fp32 (the threshold), ``degenerate`` [N] bool; the totals ``pixAcc, IoU, mIoU, mAP, mF1``; and,
    with ``pr_curve``, ``precision`` / ``recall`` over every pixel."""
    check_method(method)
    rows, means, keys = [], [], []
    P = None
    for images, labels in loader:
        gen = {"new": baselines, "lrp": lrp, "orig": orig_lrp}[_MODEL[method]]
        dev = next(gen.model.parameters()).device if gen is not None else torch.device("cuda")
        x = images.to(dev, torch.float32)
        B, H = x.shape[0], x.shape[-1]
        maps = explain(method, x, lrp, orig_lrp, baselines, is_ablation)
        if method == "full_lrp":
            grid, scale = H, 1
        else:
            grid = int(round(maps.shape[1] ** 0.5))
            scale = H // grid
        P = H * H
        r = ops.seg_metrics(maps, labels.to(dev).reshape(B, -1), grid=grid, scale=scale, thr=thr, pr_keys=pr_curve)
        packed = torch.cat([r["counts"], r["invalid"][:, None], r["degenerate"].to(torch.int64)[:, None],
                            r["ap"].view(torch.int64)[:, None], r["mean"].view(torch.int32).to(torch.int64)[:, None],
                            r["row_counts"].reshape(B, -1).to(torch.int64)], dim=1).cpu()
        bad = int(packed[:, 4].sum())
        if bad:
            raise ValueError("segmentation labels must be 0 or 1: %d other values in this batch" % bad)
        rows.append(packed)
        if pr_curve:
            keys.append(r["pr_keys"].reshape(-1))
    packed = torch.cat(rows).numpy() if rows else np.zeros((0, 8), dtype=np.int64)
    tp, fp, fn, tn = (packed[:, i] for i in range(4))
    rc = packed[:, 8:].reshape(len(tp), -1, 3)
    f1_den = 2 * rc[..., 0] + rc[..., 1] + rc[..., 2]
    with np.errstate(invalid="ignore", divide="ignore"):
        f1 = np.where(f1_den > 0, (2 * rc[..., 0]).astype(np.float64) / f1_den.astype(np.float64), 0.0)
    res = {"correct": tp + tn, "labeled": np.full(len(tp), P or 0, dtype=np.int64),
           "inter": np.stack([tn, tp], axis=1), "union": np.stack([tn + fp + fn, tp + fp + fn], axis=1),
           "ap": packed[:, 6].copy().view(np.float64), "f1": f1,
           "mean": packed[:, 7].astype(np.int32).view(np.float32), "degenerate": packed[:, 5] != 0}
    res.update(totals(res["correct"], res["labeled"], res["inter"], res["union"], res["ap"], res["f1"]))
    if pr_curve:
        if keys:
            k = torch.cat(keys)
            del keys
            ops.sort_keys(k, out=k)
            _, tps, fps = ops.pr_curve(k)
            res["precision"], res["recall"] = precision_recall(tps.cpu().numpy(), fps.cpu().numpy())
        else:
            res["precision"], res["recall"] = precision_recall([], [])
    return res


# ---- output --------------------------------------------------------------------------------------------------------------
def report_lines(results):
    """The four lines the reference prints and writes (``:325-333``)."""
    return ["Mean IoU over %d classes: %.4f\n" % (2, results["mIoU"]),
            "Pixel-wise Accuracy: %2.2f%%\n" % (results["pixAcc"] * 100),
            "Mean AP over %d classes: %.4f\n" % (2, results["mAP"]),
            "Mean F1 over %d classes: %.4f\n" % (2, results["mF1"])]


def save(results, experiment_dir, method):
    """``precision.npy`` / ``recall.npy``, ``PR_curve_{method}.png`` (when matplotlib imports) and
    ``result_mIoU_{mIoU:.4f}.txt`` with the four report lines (``:315-334``).  Returns the txt path."""
    os.makedirs(experiment_dir, exist_ok=True)
    if "precision" in results:
        np.save(os.path.join(experiment_dir, "precision.npy"), results["precision"])
        np.save(os.path.join(experiment_dir, "recall.npy"), results["recall"])
        try:
            import matplotlib
            matplotlib.use("agg")
            import matplotlib.pyplot as plt
        except ImportError:
            print("matplotlib is not installed: PR_curve_%s.png not written" % method)
        else:
            plt.figure()
            plt.plot(results["recall"], results["precision"])
            plt.savefig(os.path.join(experiment_dir, "PR_curve_{}.png".format(method)))
            plt.close()
    txt = os.path.join(experiment_dir, "result_mIoU_%.4f.txt" % results["mIoU"])
    with open(txt, "w") as fh:
        fh.writelines(report_lines(results))
    return txt


# ---- command line ----------------------------------------------------------------------------------------------------------
def build_parser():
    p = argparse.ArgumentParser(description="ImageNet-segmentation evaluation of the ViT explanation methods")
    p.add_argument("--arc", type=str, default="vgg", metavar="N", help="model architecture (names the run directory)")
    p.add_argument("--train_dataset", type=str, default="imagenet", metavar="N", help="names the run directory")
    p.add_argument("--method", type=str, required=True, choices=METHODS)
    p.add_argument("--thr", type=float, default=0., help="threshold of the PR-curve scores")
    p.add_argument("--K", type=int, default=1, help="accepted for compatibility; unused, as in the reference")
    p.add_argument("--save-img", action="store_true", default=False, help="not supported")
    for flag in ("--no-ia", "--no-fx", "--no-fgx", "--no-m", "--no-reg"):
        p.add_argument(flag, action="store_true", default=False, help="accepted for compatibility; unused")
    p.add_argument("--is-ablation", type=str2bool, default=False)
    p.add_argument("--imagenet-seg-path", type=str, required=True)
    p.add_argument("--batch-size", type=int, default=32)
    p.add_argument("--state-dict", type=str, default=None,
                   help="ViT-B/16 weights (timm key names); pretrained weights are not downloaded")
    p.add_argument("--root", type=str, default=None, help="directory holding run/ (default: the current directory)")
    return p


def parse_args(argv=None):
    p = build_parser()
    args = p.parse_args(argv)
    if args.save_img:
        p.error("--save-img is not supported")
    if args.batch_size < 1:
        p.error("--batch-size must be at least 1")
    return args


def runs_dir(args, root):
    """``run/{train_dataset}/{method}_{arc}`` (the reference's ``Saver``)."""
    return os.path.join(root, "run", args.train_dataset, args.method + "_" + args.arc)


def make_experiment_dir(runs):
    """``experiment_{n}`` (n one more than the last existing, the sorted-glob rule of ``Saver``) with the reference's empty
    ``results/{input,explain/img,explain/np}`` directories."""
    experiments = sorted(glob.glob(os.path.join(runs, "experiment_*")))
    n = int(experiments[-1].split("_")[-1]) + 1 if experiments else 0
    d = os.path.join(runs, "experiment_%d" % n)
    for sub in ("input", "explain/img", "explain/np"):
        os.makedirs(os.path.join(d, "results", sub), exist_ok=True)
    return d


def build_generators(method, state_dict=None, device="cuda", kind=None):
    """(lrp, orig_lrp, baselines) with only the façade model ``method`` needs: ``kind`` "new" (``ViT_new``), "lrp"
    (``ViT_LRP``) or "orig" (``ViT_orig_LRP``), by default the one this evaluation uses for ``method``."""
    from .baselines.ViT.ViT_explanation_generator import LRP, Baselines
    kind = kind or _MODEL[method]
    if kind == "new":
        from .baselines.ViT.ViT_new import vit_base_patch16_224 as make
    elif kind == "lrp":
        from .baselines.ViT.ViT_LRP import vit_base_patch16_224 as make
    else:
        from .baselines.ViT.ViT_orig_LRP import vit_base_patch16_224 as make
    model = make()
    if state_dict:
        model.load_state_dict(torch.load(state_dict, map_location="cpu"))
    model = model.to(device).eval()
    if kind == "new":
        return None, None, Baselines(model)
    return (LRP(model), None, None) if kind == "lrp" else (None, LRP(model), None)


def main(argv=None):
    args = parse_args(argv)
    root = args.root or os.getcwd()
    experiment_dir = make_experiment_dir(runs_dir(args, root))
    img_t, lbl_t = seg_transforms()
    ds = ImagenetSegmentation(args.imagenet_seg_path, transform=img_t, target_transform=lbl_t)
    loader = torch.utils.data.DataLoader(ds, batch_size=args.batch_size, shuffle=False, num_workers=1, drop_last=False)
    lrp, orig_lrp, baselines = build_generators(args.method, args.state_dict)
    results = segmentation_eval(args.method, loader, lrp=lrp, orig_lrp=orig_lrp, baselines=baselines, thr=args.thr,
                                is_ablation=args.is_ablation)
    save(results, experiment_dir, args.method)
    for line in report_lines(results):
        print(line)
    return results


if __name__ == "__main__":
    main()
