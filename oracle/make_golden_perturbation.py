"""Generate ``tests/golden/perturbation.npz`` by running the UNMODIFIED reference ``eval(args)`` of
``baselines/ViT/pertubation_eval_from_hdf5.py`` on CPU (authoring container).

    python -m oracle.make_golden_perturbation           # from the repo root, needs /root/reference

TEST INFRASTRUCTURE.  The script is imported from its file and run with the module globals it expects set
(``imagenet_ds``, ``sample_loader``, ``model``, ``device``); shims, none of which changes the arithmetic:
 1. ``sys.path`` gets ``baselines/ViT`` (the script imports ``ViT_explanation_generator`` / ``ViT_new`` top-level).
 2. a stub ``dataset.expl_hdf5`` module: the script imports ``ImagenetResults`` from it, and h5py may be absent; the
    samples are handed over as an in-memory dataset instead.
 3. ``args.experiment_dir`` is a temporary directory; the six ``.npy`` files ``eval`` saves are read back.

Model: a reference ``ViT_new`` at 224 x 224, patch 16, dim 64, 3 blocks, 4 heads, 10 classes, LayerNorm eps 1e-6 (the
script hard-codes ``base_size = 224 * 224``), parameters ``oracle.vit.init_params("vit_tiny_test", seed=PARAM_SEED,
rand_affine=True, img=224, patch=16)`` with the head weights x30.  12 samples in batches of 5 (the last one ragged).  Images are ``torch.rand`` and
the saliency a random permutation of 0 .. P-1 (tie-free, so the reference's ``topk`` is deterministic), both regenerated
from seeds; targets are chosen so that the first and last batch are misclassified and the middle one is classified
correctly by the unperturbed model, the pattern under which the reference's ``--wrong`` branch runs (it subtracts the
unfiltered unperturbed logits, ``:103,107``, which only broadcasts when a whole batch is kept).
Stored per mode ``{neg,pos}.{per,100}``: the six arrays; ``wrong.neg.per``: the four perturbation arrays.
"""
import argparse
import functools
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh          # noqa: E402
from oracle import vit as ovit                # noqa: E402
from oracle import perturbation as opert      # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "perturbation.npz")
KW = dict(img_size=224, patch_size=16, embed_dim=64, depth=3, num_heads=4, mlp_ratio=4., qkv_bias=True, num_classes=10)
PARAM_SEED, IMAGE_SEED, VIS_SEED, N, BATCH, EPS = 7, 11, 13, 12, 5, 1e-6
NAMES = ("model_hits", "model_dissimilarities", "perturbations_hits", "perturbations_dissimilarities",
         "perturbations_logit_diff", "perturbations_prob_diff")


def params():
    """The classifier weights are scaled x30 so that the predictions change as pixels are removed (at the init scale the
    tiny model's arg-max does not move at any step)."""
    p, heads = ovit.init_params("vit_tiny_test", seed=PARAM_SEED, rand_affine=True, img=224, patch=16)
    p["head.weight"] = p["head.weight"] * 30
    return p, heads


def samples(p=None, heads=None):
    """(images [N,3,224,224], vis [N,1,224,224], targets [N] int64), regenerated from the seeds."""
    if p is None:
        p, heads = params()
    images = torch.rand(N, 3, 224, 224, generator=torch.Generator().manual_seed(IMAGE_SEED))
    g = torch.Generator().manual_seed(VIS_SEED)
    vis = torch.stack([torch.randperm(224 * 224, generator=g).to(torch.float32) / (224 * 224) for _ in range(N)])
    vis = vis.reshape(N, 1, 224, 224)
    pred = opert.vit_logits_fn(p, heads, norm_eps=EPS)(opert.normalize(images)).argmax(1)
    target = pred.clone()
    wrong = [i for i in range(N) if i // BATCH != 1]                      # batches 0 and 2 misclassified
    target[wrong] = (pred[wrong] + 1 + torch.arange(len(wrong)) % 9) % KW["num_classes"]
    return images, vis, target


class _Samples(torch.utils.data.Dataset):
    def __init__(self, images, vis, target):
        self.t = (images, vis, target)

    def __len__(self):
        return self.t[0].shape[0]

    def __getitem__(self, i):
        return tuple(x[i] for x in self.t)


def run_reference(model, ds, neg, scale, wrong):
    ref_dir = os.path.join(rh.REF, "baselines", "ViT")
    stub = types.ModuleType("dataset.expl_hdf5")                                          # shim 2
    stub.ImagenetResults = _Samples
    pkg = types.ModuleType("dataset")
    pkg.expl_hdf5 = stub
    saved = {k: sys.modules.get(k) for k in ("dataset", "dataset.expl_hdf5")}
    sys.modules.update({"dataset": pkg, "dataset.expl_hdf5": stub})
    sys.path.insert(0, ref_dir)                                                           # shim 1
    try:
        with rh._ref_imports():
            spec = importlib.util.spec_from_file_location("pertubation_eval_from_hdf5",
                                                          os.path.join(ref_dir, "pertubation_eval_from_hdf5.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            mod.imagenet_ds = ds
            mod.sample_loader = torch.utils.data.DataLoader(ds, batch_size=BATCH, shuffle=False)
            mod.model = model
            mod.device = torch.device("cpu")
            with tempfile.TemporaryDirectory() as d:                                     # shim 3
                mod.eval(argparse.Namespace(neg=neg, scale=scale, wrong=wrong, experiment_dir=d))
                return {n: np.load(os.path.join(d, n + ".npy")) for n in NAMES}
    finally:
        sys.path.remove(ref_dir)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def main():
    import torch.nn as nn
    p, heads = params()
    images, vis, target = samples(p, heads)
    model = rh.build_vit_new("custom", state_dict=p, norm_layer=functools.partial(nn.LayerNorm, eps=EPS), **KW)
    ds = _Samples(images, vis, target)
    out = {"param_seed": np.int64(PARAM_SEED), "image_seed": np.int64(IMAGE_SEED), "vis_seed": np.int64(VIS_SEED),
           "n": np.int64(N), "batch": np.int64(BATCH), "target": target.numpy(),
           "image_checksum": images.double().sum(dim=(1, 2, 3)).numpy(), "vis_checksum": vis.double().sum(dim=(1, 2, 3)).numpy()}
    with torch.no_grad():
        for neg in (True, False):
            for scale in ("per", "100"):
                r = run_reference(model, ds, neg, scale, False)
                for n in NAMES:
                    out["%s.%s.%s" % ("neg" if neg else "pos", scale, n)] = r[n]
        r = run_reference(model, ds, True, "per", True)
        for n in NAMES[2:]:
            out["wrong.neg.per." + n] = r[n]
    np.savez_compressed(OUT, **out)
    print("perturbation.npz", len(out), "arrays; model hits", out["neg.per.model_hits"],
          "perturbation hits per step", out["neg.per.perturbations_hits"].mean(1), out["pos.per.perturbations_hits"].mean(1))


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
