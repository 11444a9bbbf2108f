"""Positive / negative perturbation evaluation of saved explanations (``baselines/ViT/pertubation_eval_from_hdf5.py``).

Reads the ``results.hdf5`` that ``hdf5_writer.compute_saliency_and_save`` writes and measures how fast the classifier's
accuracy falls as the most relevant (positive) or least relevant (negative, ``neg=True``) pixels are removed in nine
steps — the number the paper reports per method.  Per data batch: one ``te_perturb_images`` call builds the unperturbed
and the nine perturbed, normalised inputs, the engine runs their forwards, one ``te_logit_stats`` call reduces the logits,
and the results come back in one device-to-host copy.

    python -m transformer_explainability_b200.perturbation --method transformer_attribution --neg True \\
        --state-dict vit_base_patch16_224.pth

Deviations from the reference script (DESIGN.md §1):
 * the pixels removed at a step are the first ``k`` in the order NaN, descending value, ascending pixel index; the
   reference's ``torch.topk`` leaves the choice among tied values to its implementation;
 * ``--neg`` / ``--is-ablation`` parse real booleans (the reference's ``type=bool`` turns ``--neg False`` into True);
 * with ``--wrong`` the model arrays hold one entry per sample in dataset order (the reference advances its model index by
   the filtered count and overwrites ``model_hits.npy`` out of place), and the differences are taken against the
   unperturbed outputs of the kept samples (the reference subtracts the whole batch's, which only broadcasts when every
   sample of the batch is kept);
 * the CLI also prints the area under the hits curve over ``[0, steps...]`` (trapezoid rule), which the reference does not.
"""
import argparse
import glob
import os
import struct

import numpy as np
import torch

from . import ops

STEPS = {"per": (224 * 224, [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]),
         "100": (100, [5, 10, 15, 20, 25, 30, 35, 40, 45])}
NAMES = ("model_hits", "model_dissimilarities", "perturbations_hits", "perturbations_dissimilarities",
         "perturbations_logit_diff", "perturbations_prob_diff")


def perturbation_steps(scale):
    """(steps, pixel counts): ``int(base_size * step)`` in Python double, as the reference computes them."""
    if scale not in STEPS:
        raise ValueError("scale not valid: %r (expected 'per' or '100')" % (scale,))
    base_size, steps = STEPS[scale]
    return list(steps), [int(base_size * s) for s in steps]


# ---- the results file --------------------------------------------------------------------------------------------------
def _minimal_hdf5_layout(path):
    """{name: (shape, numpy dtype, byte offset)} of the contiguous datasets of a file written by
    ``hdf5_writer.write_minimal_hdf5``, read from the headers only (the same walk as ``read_minimal_hdf5``)."""
    from .hdf5_writer import _SIG
    with open(path, "rb") as f:
        def at(off, n):
            f.seek(off)
            return f.read(n)
        if at(0, 8) != _SIG:
            raise ValueError("%s: not an HDF5 file" % path)
        _, root_hdr, _, _, btree, heap = struct.unpack("<QQIIQQ", at(56, 40))
        if at(heap, 4) != b"HEAP" or at(btree, 4) != b"TREE":
            raise ValueError("%s: not the contiguous layout of the built-in writer (install h5py to read it)" % path)
        hdata = struct.unpack("<Q", at(heap + 24, 8))[0]
        snod = struct.unpack("<Q", at(btree + 32, 8))[0]
        if at(snod, 4) != b"SNOD":
            raise ValueError("%s: unexpected group layout (install h5py to read it)" % path)
        nsym = struct.unpack("<H", at(snod + 6, 2))[0]
        out = {}
        for i in range(nsym):
            noff, ohdr = struct.unpack("<QQ", at(snod + 8 + 40 * i, 16))
            name = at(hdata + noff, 256).split(b"\0", 1)[0].decode("ascii")
            _, _, nmsg, _, hsize = struct.unpack("<BBHII", at(ohdr, 12))
            body = at(ohdr + 16, hsize)
            pos, shape, dtype, addr, layout = 0, None, None, None, None
            for _ in range(nmsg):
                mt, ms = struct.unpack_from("<HH", body, pos)
                d = pos + 8
                if mt == 0x0001:
                    shape = struct.unpack_from("<%dQ" % body[d + 1], body, d + 8)
                elif mt == 0x0003:
                    cls, tsize = body[d] & 0x0F, struct.unpack_from("<I", body, d + 4)[0]
                    dtype = {(1, 4): np.dtype("<f4"), (0, 4): np.dtype("<i4")}.get((cls, tsize))
                elif mt == 0x0008:
                    lv, layout, addr, _ = struct.unpack_from("<BBQQ", body, d)
                pos = d + ms
            if dtype is None or layout != 1 or shape is None:
                raise ValueError("%s: dataset %r is not a contiguous float32 / int32 array (install h5py to read it)"
                                 % (path, name))
            out[name] = (tuple(int(s) for s in shape), dtype, addr)
        return out


class ImagenetResults(torch.utils.data.Dataset):
    """Drop-in for the reference's ``dataset/expl_hdf5.py``: ``ImagenetResults(method_dir)[i]`` -> (image [3,H,W], vis
    [1,H,W], target int64) from ``method_dir/results.hdf5``.  Uses h5py when it can be imported; otherwise reads the
    contiguous layout the built-in writer emits, lazily per item through ``np.memmap`` (the whole ImageNet-val file is
    about 40 GB)."""

    def __init__(self, path):
        super().__init__()
        self.path = os.path.join(path, "results.hdf5")
        self.data = None
        try:
            import h5py
            self._layout = None
        except ImportError:
            h5py = None
            self._layout = _minimal_hdf5_layout(self.path)
            if not {"image", "vis", "target"} <= set(self._layout):
                raise ValueError("%s: image / vis / target datasets expected" % self.path)
        if h5py is not None:
            with h5py.File(self.path, "r") as f:
                self.data_length = len(f["/image"])
        else:
            self.data_length = self._layout["image"][0][0]

    def __len__(self):
        return self.data_length

    def __getitem__(self, item):
        if self.data is None:
            if self._layout is None:
                import h5py
                self.data = h5py.File(self.path, "r")
            else:
                self.data = {n: np.memmap(self.path, dtype=dt, mode="r", offset=off, shape=shape)
                             for n, (shape, dt, off) in self._layout.items()}
        image = torch.tensor(np.array(self.data["image"][item]))
        vis = torch.tensor(np.array(self.data["vis"][item]))
        target = torch.tensor(np.array(self.data["target"][item])).long()
        return image, vis, target

    def __getstate__(self):                      # DataLoader workers open the file themselves
        state = dict(self.__dict__)
        state["data"] = None
        return state


# ---- the evaluation ------------------------------------------------------------------------------------------------------
def _forward(eng, x, chunk):
    """Engine forwards of x [R,C,H,W] in chunks of at most ``chunk`` rows -> logits [R, classes]."""
    R = x.shape[0]
    n = -(-R // chunk)
    step = -(-R // n)                             # near-equal chunks rather than a small ragged tail
    return torch.cat([eng.forward(x[s:s + step]) for s in range(0, R, step)])


def perturbation_eval(model, loader, neg=True, scale="per", wrong=False, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5),
                      chunk=None):
    """``eval(args)`` of ``pertubation_eval_from_hdf5.py`` on the engine of ``model`` (a ``ViT_new`` / ``ViT_LRP`` façade
    model, with its engine flags).  ``loader`` yields (image [B,C,H,W] in [0, 1], vis [B,1,H,W], target [B]).  Returns the
    six float64 arrays the reference saves: ``model_hits`` / ``model_dissimilarities`` [N] and
    ``perturbations_{hits,dissimilarities,logit_diff,prob_diff}`` [9, n].  ``chunk``: rows per engine forward (default:
    ``ViTEngine.max_chunk``)."""
    eng = model.engine()
    dev = eng.device
    _, ks = perturbation_steps(scale)
    S = len(ks)
    model_rows, pert_rows = [], []
    for data, vis, target in loader:
        x = data.to(dev, torch.float32).contiguous()
        s = vis.to(dev, torch.float32).reshape(x.shape[0], -1).contiguous()
        t = target.to(dev).reshape(-1).to(torch.int32)
        B = x.shape[0]
        c = chunk or eng.max_chunk(limit=(S + 1) * B)
        if not wrong:
            xs = ops.perturb_images(x, s, [0] + ks, negate=neg, mean=mean, std=std)           # [S+1,B,C,H,W]
            logits = _forward(eng, xs.reshape((S + 1) * B, *x.shape[1:]), c)
            pred, ml, mp, dis = (u.reshape(S + 1, B) for u in ops.logit_stats(logits, t.repeat(S + 1)))
            hits = (pred == t).to(torch.float32)
            res = torch.cat([torch.stack([hits[0], dis[0]]), hits[1:], dis[1:], ml[1:] - ml[0], mp[1:] - mp[0]]).cpu()
            model_rows.append(res[:2])
            pert_rows.append(res[2:].reshape(4, S, B))
            continue
        x0 = ops.perturb_images(x, s, [0], negate=neg, mean=mean, std=std)[0]
        pred0, ml0, mp0, dis0 = ops.logit_stats(_forward(eng, x0, c), t)
        head = torch.stack([(pred0 == t).to(torch.float32), dis0]).cpu()                      # the extra sync of --wrong
        model_rows.append(head)
        wid = torch.nonzero(head[0] == 0).flatten().to(dev)
        if len(wid) == 0:
            continue
        xw, sw, tw = x.index_select(0, wid).contiguous(), s.index_select(0, wid).contiguous(), t.index_select(0, wid)
        n = len(wid)
        xs = ops.perturb_images(xw, sw, ks, negate=neg, mean=mean, std=std)
        pred, ml, mp, dis = (u.reshape(S, n) for u in ops.logit_stats(_forward(eng, xs.reshape(S * n, *x.shape[1:]), c),
                                                                        tw.repeat(S)))
        res = torch.cat([(pred == tw).to(torch.float32), dis, ml - ml0[wid], mp - mp0[wid]]).cpu()
        pert_rows.append(res.reshape(4, S, n))
    model = torch.cat(model_rows, dim=1).double().numpy() if model_rows else np.zeros((2, 0))
    pert = torch.cat(pert_rows, dim=2).double().numpy() if pert_rows else np.zeros((4, S, 0))
    return {"model_hits": model[0], "model_dissimilarities": model[1], "perturbations_hits": pert[0],
            "perturbations_dissimilarities": pert[1], "perturbations_logit_diff": pert[2], "perturbations_prob_diff": pert[3]}


def hits_auc(results, scale="per"):
    """Area under the mean-hits curve over x = [0, steps...] (trapezoid rule): the unperturbed accuracy at 0, then the
    accuracy after each step; the steps are 0.1 ... 0.9 (fraction of the 224 x 224 pixels) for ``scale="per"`` and
    5 ... 45 (hundreds of pixels) for ``scale="100"``.  Not in the reference script."""
    steps, _ = perturbation_steps(scale)
    xs = [0.0] + [float(v) for v in steps]
    hits = results["perturbations_hits"]
    model_hits = results["model_hits"]
    ys = [float(np.mean(model_hits)) if len(model_hits) else float("nan")] + \
         [float(np.mean(hits[i])) if hits.shape[1] else float("nan") for i in range(hits.shape[0])]
    return float(sum((xs[i + 1] - xs[i]) * (ys[i] + ys[i + 1]) / 2 for i in range(len(xs) - 1)))


def save(results, experiment_dir):
    """The six ``.npy`` files of the reference (``pertubation_eval_from_hdf5.py:123-128``)."""
    os.makedirs(experiment_dir, exist_ok=True)
    for n in NAMES:
        np.save(os.path.join(experiment_dir, n + ".npy"), results[n])


# ---- command line ----------------------------------------------------------------------------------------------------------
def str2bool(v):
    if isinstance(v, bool):
        return v
    s = str(v).strip().lower()
    if s in ("1", "true", "t", "yes", "y", "on"):
        return True
    if s in ("0", "false", "f", "no", "n", "off"):
        return False
    raise argparse.ArgumentTypeError("boolean expected, got %r" % (v,))


METHODS = ['rollout', 'lrp', 'transformer_attribution', 'full_lrp', 'v_gradcam', 'lrp_last_layer', 'lrp_second_layer',
           'gradcam', 'attn_last_layer', 'attn_gradcam', 'input_grads',
           'attn_grad_rollout']      # the LRP-free gradient-weighted attention rollout (Chefer, Gur, Wolf, ICCV 2021)


def build_parser():
    p = argparse.ArgumentParser(description="Positive / negative perturbation evaluation of saved explanations")
    p.add_argument("--batch-size", type=int, default=16)
    p.add_argument("--neg", type=str2bool, default=True)
    p.add_argument("--value", action="store_true", default=False)
    p.add_argument("--scale", type=str, default="per", choices=["per", "100"])
    p.add_argument("--method", type=str, default="grad_rollout", choices=METHODS)
    p.add_argument("--vis-class", type=str, default="top", choices=["top", "target", "index"])
    p.add_argument("--wrong", action="store_true", default=False)
    p.add_argument("--class-id", type=int, default=0)
    p.add_argument("--is-ablation", type=str2bool, default=False)
    p.add_argument("--state-dict", type=str, default=None,
                   help="ViT-B/16 weights (timm key names); pretrained weights are not downloaded")
    p.add_argument("--root", type=str, default=None,
                   help="directory holding visualizations/ and experiments/ (default: the current directory)")
    return p


def _fold(args):
    if args.vis_class == "index":
        return "%s_%d" % (args.vis_class, args.class_id)
    return os.path.join(args.vis_class, "ablation" if args.is_ablation else "not_ablation")


def runs_dir(args, root):
    """``experiments/perturbations/{method}_{neg|pos}/{vis_class}/{ablation|not_ablation}`` (+ ``_wrong``), or
    ``.../{vis_class}_{class_id}`` for ``--vis-class index``."""
    exp_name = args.method + ("_neg" if args.neg else "_pos")
    d = os.path.join(root, "experiments", "perturbations", exp_name, _fold(args))
    return d + "_wrong" if args.wrong else d


def next_experiment_dir(runs):
    """``experiment_{n}`` with n one more than the last existing one (the reference's sorted-glob rule)."""
    experiments = sorted(glob.glob(os.path.join(runs, "experiment_*")))
    n = int(experiments[-1].split("_")[-1]) + 1 if experiments else 0
    return os.path.join(runs, "experiment_%d" % n)


def vis_method_dir(args, root):
    return os.path.join(root, "visualizations", args.method, _fold(args))


def report(results, scale):
    """What the reference prints (``:130-134``) and the area under the hits curve."""
    steps, _ = perturbation_steps(scale)
    print(np.mean(results["model_hits"]), np.std(results["model_hits"]))
    print(np.mean(results["model_dissimilarities"]), np.std(results["model_dissimilarities"]))
    print(steps)
    print(np.mean(results["perturbations_hits"], axis=1), np.std(results["perturbations_hits"], axis=1))
    print(np.mean(results["perturbations_dissimilarities"], axis=1), np.std(results["perturbations_dissimilarities"], axis=1))
    print("hits AUC", hits_auc(results, scale))


def main(argv=None):
    args = build_parser().parse_args(argv)
    root = args.root or os.getcwd()
    print(args.method + ("_neg" if args.neg else "_pos"))
    experiment_dir = next_experiment_dir(runs_dir(args, root))
    from .baselines.ViT.ViT_new import vit_base_patch16_224
    model = vit_base_patch16_224()
    if args.state_dict:
        model.load_state_dict(torch.load(args.state_dict, map_location="cpu"))
    model = model.cuda().eval()
    ds = ImagenetResults(vis_method_dir(args, root))
    loader = torch.utils.data.DataLoader(ds, batch_size=args.batch_size, num_workers=2, shuffle=False)
    results = perturbation_eval(model, loader, neg=args.neg, scale=args.scale, wrong=args.wrong)
    save(results, experiment_dir)
    report(results, args.scale)
    return results


if __name__ == "__main__":
    main()
