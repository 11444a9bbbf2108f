"""Generate ``tests/golden/segmentation.npz`` by running the UNMODIFIED reference ``baselines/ViT/imagenet_seg_eval.py``
on CPU for each of its six working methods (authoring container).

    python -m oracle.make_golden_segmentation           # from the repo root, needs /root/reference and sklearn

TEST INFRASTRUCTURE.  The script does all its work at import time; it is executed from its file with these shims, none
of which changes the arithmetic:
 1. ``sys.argv`` carries ``--method`` / ``--imagenet-seg-path``; the working directory is a temporary directory (the
    script's ``Saver`` writes ``run/imagenet/...`` relative to it); ``rh._cpu_cuda_shim`` makes ``.cuda()`` a no-op.
 2. a stub ``data.Imagenet`` module whose ``Imagenet_Segmentation`` serves the seeded PIL images and masks below through
    the transforms the script passes (the real one needs h5py and the .mat file).
 3. stub ``imageio``, ``matplotlib.pyplot`` and ``utils.render`` modules (only used for ``--save-img`` and the PR plot).
 4. the three ``vit_base_patch16_224`` factories return the tiny model below; ``pretrained`` is ignored.
 5. recording wrappers around ``utils.metrices``' four metric functions and the generator methods; they record their
    results (the per-sample counts, AP, F1 and the raw maps) and return them unchanged.
After the run the module globals ``pixAcc, IoU, mIoU, mAp, mF1`` are read back, and ``precision.npy`` / ``recall.npy`` from
the experiment directory (stored as ``oracle.segmentation.pr_summary``).

Model: the 224 / 16 ViT of ``make_golden_perturbation`` (dim 64, 3 blocks, 4 heads, 10 classes, LayerNorm eps 1e-6) with
its parameter seed but without the x30 head scaling (with it, every attention-GradCAM map of these samples is constant and
the script fails on the NaN), for all three model files.  Samples: ``N`` seeded RGB images of different sizes (so the script's own
Resize runs) with seeded elliptic blob masks; mask 2 is all 0 and mask 5 all 1.  ``full_lrp`` runs on sample 1 only
(``SUBSETS``): its map is stored per pixel (224 x 224 fp32, which hardly compresses), and one keeps the fixture small.
"""
import contextlib
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

from oracle import ref_harness as rh                  # noqa: E402
from oracle import make_golden_perturbation as mgp    # noqa: E402
from oracle import segmentation as oseg               # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "segmentation.npz")
METHODS = ("rollout", "transformer_attribution", "full_lrp", "lrp_last_layer", "attn_last_layer", "attn_gradcam")
SIZES = [(224, 224), (300, 260), (180, 240), (257, 199), (224, 320), (150, 150), (333, 224), (240, 180)]   # (h, w)
N = len(SIZES)
SAMPLE_SEED = 31
EMPTY_MASK, FULL_MASK = 2, 5
SUBSETS = {"full_lrp": (1,)}        # sample indices the script runs on per method (default: all)


def method_samples(method):
    return list(SUBSETS.get(method, range(N)))


def params():
    from oracle import vit as ovit
    p, heads = ovit.init_params("vit_tiny_test", seed=mgp.PARAM_SEED, rand_affine=True, img=224, patch=16)
    return p, heads


def raw_samples():
    """[(uint8 image [h,w,3], uint8 mask [h,w] of 0 / 1)] regenerated from the seed."""
    g = np.random.default_rng(SAMPLE_SEED)
    out = []
    for i, (h, w) in enumerate(SIZES):
        img = g.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        yy, xx = np.mgrid[0:h, 0:w]
        mask = np.zeros((h, w), dtype=np.uint8)
        for _ in range(int(g.integers(1, 4))):
            cy, cx = g.uniform(0.2, 0.8) * h, g.uniform(0.2, 0.8) * w
            ry, rx = g.uniform(0.1, 0.35) * h, g.uniform(0.1, 0.35) * w
            mask |= (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1).astype(np.uint8)
        if i == EMPTY_MASK:
            mask[:] = 0
        if i == FULL_MASK:
            mask[:] = 1
        out.append((img, mask))
    return out


class SegmentationSamples(torch.utils.data.Dataset):
    """The stub ``Imagenet_Segmentation``: ``data/Imagenet.py:59-77`` on in-memory arrays."""

    def __init__(self, path=None, transform=None, target_transform=None, indices=None):
        raw = raw_samples()
        self.samples = raw if indices is None else [raw[i] for i in indices]
        self.transform = transform
        self.target_transform = target_transform

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, index):
        from PIL import Image
        img, target = self.samples[index]
        img = Image.fromarray(img).convert('RGB')
        target = Image.fromarray(target)
        if self.transform is not None:
            img = self.transform(img)
        if self.target_transform is not None:
            target = np.array(self.target_transform(target)).astype('int32')
            target = torch.from_numpy(target).long()
        return img, target


def samples():
    """(images [N,3,224,224] normalised as the script does, labels [N,224,224] int64) through ``seg_transforms``."""
    from transformer_explainability_b200.segmentation import seg_transforms
    img_t, lbl_t = seg_transforms()
    ds = SegmentationSamples(transform=img_t, target_transform=lbl_t)
    items = [ds[i] for i in range(len(ds))]
    return torch.stack([x for x, _ in items]), torch.stack([y for _, y in items])


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    return m


@contextlib.contextmanager
def _swapped_modules(mods):
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def run_reference(method, p):
    """Run the script for ``method`` on ``method_samples(method)``; returns (records, module globals, precision,
    recall)."""
    import torch.nn as nn
    ref_dir = os.path.join(rh.REF, "baselines", "ViT")
    rec = {"maps": [], "pix": [], "iu": [], "ap": [], "f1": []}
    plt = _stub("matplotlib.pyplot", switch_backend=lambda *a, **k: None, figure=lambda *a, **k: None,
                plot=lambda *a, **k: None, savefig=lambda *a, **k: None)
    stubs = {"data": _stub("data"), "data.Imagenet": _stub("data.Imagenet", Imagenet_Segmentation=functools.partial(
                 SegmentationSamples, indices=method_samples(method))),
             "imageio": _stub("imageio", imsave=lambda *a, **k: None), "matplotlib": _stub("matplotlib", pyplot=plt),
             "matplotlib.pyplot": plt, "utils.render": _stub("utils.render")}
    stubs["data"].Imagenet = stubs["data.Imagenet"]
    own = [k for k in sys.modules if k == "utils" or k.startswith("utils.")]
    saved_utils = {k: sys.modules.pop(k) for k in own}
    old_cwd, old_argv = os.getcwd(), sys.argv
    sys.path.insert(0, ref_dir)
    try:
        with rh._ref_imports(), _swapped_modules(stubs), tempfile.TemporaryDirectory() as tmp, rh._cpu_cuda_shim():
            import utils
            import utils.metrices as metrices
            utils.render = stubs["utils.render"]
            import ViT_explanation_generator as gen
            import ViT_new
            import ViT_LRP
            import ViT_orig_LRP
            eps_ln = functools.partial(nn.LayerNorm, eps=mgp.EPS)

            def factory(mod, **extra):
                def make(pretrained=False, **kw):
                    m = mod.VisionTransformer(**mgp.KW, **extra)
                    m.load_state_dict(p)
                    return m
                return make
            ViT_new.vit_base_patch16_224 = factory(ViT_new, norm_layer=eps_ln)
            ViT_LRP.vit_base_patch16_224 = factory(ViT_LRP)
            ViT_orig_LRP.vit_base_patch16_224 = factory(ViT_orig_LRP)

            def recorder(key, fn, conv=lambda r: r):
                @functools.wraps(fn)
                def wrapped(*a, **k):
                    r = fn(*a, **k)
                    rec[key].append(conv(r))
                    return r
                return wrapped
            for cls, name in ((gen.LRP, "generate_LRP"), (gen.Baselines, "generate_rollout"),
                              (gen.Baselines, "generate_cam_attn")):
                setattr(cls, name, recorder("maps", getattr(cls, name), lambda r: r.detach().clone().reshape(-1)))
            orig = {n: getattr(metrices, n) for n in ("batch_pix_accuracy", "batch_intersection_union", "get_ap_scores",
                                                       "get_f1_scores")}
            metrices.batch_pix_accuracy = recorder("pix", orig["batch_pix_accuracy"])
            metrices.batch_intersection_union = recorder("iu", orig["batch_intersection_union"])
            metrices.get_ap_scores = recorder("ap", orig["get_ap_scores"])
            metrices.get_f1_scores = recorder("f1", orig["get_f1_scores"])
            os.chdir(tmp)
            sys.argv = ["imagenet_seg_eval.py", "--method", method, "--imagenet-seg-path", "unused.mat"]
            try:
                spec = importlib.util.spec_from_file_location("imagenet_seg_eval", os.path.join(ref_dir, "imagenet_seg_eval.py"))
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
                for n, f in orig.items():
                    setattr(metrices, n, f)
                exp = mod.saver.experiment_dir
                precision = np.load(os.path.join(exp, "precision.npy"))
                recall = np.load(os.path.join(exp, "recall.npy"))
                glob = {k: getattr(mod, k) for k in ("pixAcc", "IoU", "mIoU", "mAp", "mF1")}
                txt = [f for f in os.listdir(exp) if f.startswith("result_mIoU_")]
                with open(os.path.join(exp, txt[0])) as fh:
                    glob["txt_name"], glob["txt"] = txt[0], fh.read()
            finally:
                os.chdir(old_cwd)
                sys.argv = old_argv
            for k in ("ViT_explanation_generator", "ViT_new", "ViT_LRP", "ViT_orig_LRP"):
                sys.modules.pop(k, None)
            for k in [k for k in sys.modules if k == "utils" or k.startswith("utils.")]:
                sys.modules.pop(k)
    finally:
        sys.path.remove(ref_dir)
        sys.modules.update(saved_utils)
    return rec, glob, precision, recall


def main():
    import sklearn
    p, _ = params()
    images, labels = samples()
    out = {"n": np.int64(N), "sklearn_version": np.array(sklearn.__version__),
           "image_checksum": images.double().sum(dim=(1, 2, 3)).numpy(),
           "labels": labels.numpy().astype(np.uint8), "empty_mask": np.int64(EMPTY_MASK), "full_mask": np.int64(FULL_MASK)}
    for method in METHODS:
        rec, glob, precision, recall = run_reference(method, p)
        n = len(method_samples(method))
        assert len(rec["maps"]) == n and len(rec["pix"]) == n, (method, len(rec["maps"]), len(rec["pix"]))
        pre = method + "."
        out[pre + "samples"] = np.array(method_samples(method), dtype=np.int64)
        out[pre + "maps"] = torch.stack(rec["maps"]).to(torch.float32).numpy()
        out[pre + "correct"] = np.array([int(c) for c, _ in rec["pix"]], dtype=np.int64)
        out[pre + "labeled"] = np.array([int(l) for _, l in rec["pix"]], dtype=np.int64)
        out[pre + "inter"] = np.stack([np.asarray(i, dtype=np.int64) for i, _ in rec["iu"]])
        out[pre + "union"] = np.stack([np.asarray(u, dtype=np.int64) for _, u in rec["iu"]])
        out[pre + "ap"] = np.array([float(np.nan_to_num(a)[0]) for a in rec["ap"]])
        out[pre + "f1"] = np.stack([np.nan_to_num(np.asarray(f, dtype=np.float64)) for f in rec["f1"]])   # [n, rows]
        for k in ("pixAcc", "mIoU", "mAp", "mF1"):
            out[pre + k] = np.float64(glob[k])
        out[pre + "IoU"] = np.asarray(glob["IoU"], dtype=np.float64)
        out[pre + "txt_name"] = np.array(glob["txt_name"])
        out[pre + "txt"] = np.array(glob["txt"])
        for k, v in oseg.pr_summary(precision, recall).items():
            out[pre + k] = v
        print(method, "pixAcc %.4f mIoU %.4f mAP %.4f mF1 %.4f PR points %d" % (glob["pixAcc"], glob["mIoU"], glob["mAp"],
                                                                               glob["mF1"], len(precision)))
    np.savez_compressed(OUT, **out)
    print("segmentation.npz", len(out), "arrays,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
