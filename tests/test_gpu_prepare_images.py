"""GPU: ``ops.prepare_images`` (te_prepare_images) against torchvision's CPU ``Resize((224, 224)) + ToTensor()``, and the
generate_visualizations command (``python -m transformer_explainability_b200.hdf5_writer``) end to end.

* One ragged batch of about 40 images (ImageNet-val sizes, extreme aspect ratios, upscaling, 1 x 1, an image tall enough
  for Pillow to resize vertically first, JPEG round trips, grayscale / CMYK / palette / RGBA sources converted to RGB) is
  ``torch.equal`` to torchvision's CPU transform, and the normalised output to ``hdf5_writer.normalize`` of it.
* Each image prepared alone gives the bits it gets in the batch.
* Outputs and workspace pre-filled with 0xFF and 0x5A (as in test_gpu_poison.py) give identical bits and guards.
* The command on a synthetic ImageNet tree (11 JPEGs in 3 classes, batch 4 with a ragged last batch, seeded random-init
  ViT-B weights) writes ``results.hdf5`` whose ``image`` / ``target`` / ``vis`` are bit-identical to
  ``compute_saliency_and_save`` fed by a torchvision CPU-transform DataLoader over the same folder, for every method and
  ``--vis-class`` top / target; the perturbation command then reads that directory and writes its six arrays.
"""
import ctypes
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from transformer_explainability_b200 import _lib, hdf5_writer, ops, perturbation, segmentation

pytestmark = pytest.mark.gpu

SIZES = [(375, 500), (500, 375), (500, 333), (333, 500), (500, 500), (1200, 801), (801, 1200), (1024, 1365), (224, 224),
         (224, 300), (300, 224), (100, 150), (57, 999), (999, 57), (1, 1), (1, 500), (500, 1), (2, 3), (4096, 7),
         (1500, 9), (701, 7), (448, 448), (223, 225), (16, 16)]


def _smooth(h, w, rng):
    """A photo-like image: smooth gradients plus noise (so JPEG keeps some structure)."""
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * 255 // max(w - 1, 1)), (y * 255 // max(h - 1, 1)), ((x + y) * 127 // max(h + w - 2, 1))], -1)
    return np.clip(base + rng.integers(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)


def _jpeg(img, **kw):
    buf = io.BytesIO()
    img.save(buf, format="JPEG", **kw)
    buf.seek(0)
    return Image.open(buf).convert("RGB")


def corpus():
    """~40 RGB PIL images, as the reader would hand them over."""
    rng = np.random.default_rng(0)
    imgs = [Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)) for h, w in SIZES]
    for h, w in ((375, 500), (500, 333), (333, 500), (480, 640), (1200, 801), (64, 900)):
        imgs.append(_jpeg(Image.fromarray(_smooth(h, w, rng)), quality=85))
    gray = Image.fromarray(_smooth(400, 300, rng)[..., 0])
    imgs.append(gray.convert("RGB"))                                            # grayscale source
    imgs.append(_jpeg(gray, quality=90))                                        # grayscale JPEG
    imgs.append(_jpeg(Image.fromarray(_smooth(350, 420, rng)).convert("CMYK"), quality=90))    # CMYK JPEG
    imgs.append(Image.fromarray(_smooth(300, 310, rng)).convert("P").convert("RGB"))          # palette source
    rgba = np.concatenate([_smooth(250, 260, rng), rng.integers(0, 256, (250, 260, 1), dtype=np.uint8)], -1)
    imgs.append(Image.fromarray(rgba, "RGBA").convert("RGB"))
    imgs.append(Image.fromarray(_smooth(20, 30, rng)))                          # upscaling, smooth
    for im in imgs:
        assert im.mode == "RGB"
    return imgs


def reference(imgs, out_hw=(224, 224)):
    import torchvision.transforms as T
    t = T.Compose([T.Resize(out_hw), T.ToTensor()])
    return torch.stack([t(im) for im in imgs])


def packed(imgs):
    p, sizes, offsets, _ = hdf5_writer.pack_images([(np.array(im), 0) for im in imgs])
    return p.cuda(), sizes.numpy(), offsets.numpy()


@pytest.fixture(scope="module")
def images():
    return corpus()


@pytest.mark.parametrize("out_hw", [(224, 224), (100, 384)])
def test_batch_equals_torchvision(images, out_hw):
    assert len(images) >= 36
    p, sizes, offsets = packed(images)
    out01, out_norm = ops.prepare_images(p, sizes, offsets, out_hw, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5))
    ref = reference(images, out_hw)
    assert out01.shape == ref.shape and out01.dtype == torch.float32
    bad = [i for i in range(len(images)) if not torch.equal(out01[i].cpu(), ref[i])]
    assert not bad, "images %s differ from torchvision (sizes %s)" % (bad, [images[i].size for i in bad])
    assert torch.equal(out_norm, hdf5_writer.normalize(out01))
    other, none = ops.prepare_images(p, sizes, offsets, out_hw)
    assert none is None and torch.equal(other, out01)


def test_each_image_alone_equals_batch(images):
    p, sizes, offsets = packed(images)
    batch, _ = ops.prepare_images(p, sizes, offsets)
    for i, im in enumerate(images):
        q, s, o = packed([im])
        alone, _ = ops.prepare_images(q, s, o)
        assert torch.equal(alone[0], batch[i]), i
    # the same images packed in reverse order, with gaps between them
    rev = images[::-1]
    arrays = [np.array(im).reshape(-1) for im in rev]
    offs, pos = [], 0
    for a in arrays:
        pos += 17
        offs.append(pos)
        pos += a.size
    buf = np.zeros(pos + 5, np.uint8)
    for a, o in zip(arrays, offs):
        buf[o:o + a.size] = a
    out, _ = ops.prepare_images(torch.from_numpy(buf).cuda(), [im.size[::-1] for im in rev], offs)
    assert torch.equal(out, batch.flip(0))


GUARD = 1 << 20


def _raw_call(p, sizes, offsets, pattern):
    """te_prepare_images on outputs and a workspace allocated with a guard and pre-filled with ``pattern`` (None: torch's
    allocator as it comes)."""
    lib = _lib.load()
    B, oh, ow = len(sizes), 224, 224
    nbytes = lib.te_prepare_images_workspace_bytes(B, int(sizes[:, 0].max()), int(sizes[:, 1].max()), oh, ow)
    assert nbytes > 0
    n_out = B * 3 * oh * ow * 4

    def buf(n):
        b = torch.empty(n + GUARD, dtype=torch.uint8, device="cuda")
        if pattern is not None:
            b.fill_(pattern)
        return b
    o01, onorm, ws = buf(n_out), buf(n_out), buf(nbytes)
    mean = (ctypes.c_float * 3)(0.485, 0.456, 0.406)
    std = (ctypes.c_float * 3)(0.229, 0.224, 0.225)
    sz = np.ascontiguousarray(sizes, np.int32)
    off = np.ascontiguousarray(offsets, np.int64)
    r = lib.te_prepare_images(_lib.ptr(p), p.numel(), B, sz.ctypes.data_as(ctypes.c_void_p), off.ctypes.data_as(ctypes.c_void_p),
                              oh, ow, mean, std, _lib.ptr(o01), _lib.ptr(onorm), _lib.ptr(ws), nbytes,
                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert r == 0, lib.te_last_error()
    torch.cuda.synchronize()
    return o01, onorm, n_out


def test_poisoned_outputs_and_workspace(images):
    p, sizes, offsets = packed(images)
    base = None
    for pattern in (None, 0xFF, 0x5A):
        o01, onorm, n = _raw_call(p, sizes, offsets, pattern)
        got = (o01[:n].clone(), onorm[:n].clone())
        if base is None:
            base = got
            assert torch.equal(got[0].view(torch.float32).reshape(len(images), 3, 224, 224).cpu(), reference(images))
        else:
            assert torch.equal(got[0], base[0]) and torch.equal(got[1], base[1]), pattern
            assert bool((o01[n:] == pattern).all()) and bool((onorm[n:] == pattern).all()), pattern


# ---- the command end to end ----------------------------------------------------------------------------------------------
N_IMAGES = 11
WNIDS = ("n01440764", "n01443537", "n01484850")


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """A synthetic ImageNet validation folder (meta.bin + val/{wnid}/*.JPEG, one grayscale and one CMYK JPEG among them)
    and seeded random-init ViT-B weights."""
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224
    root = str(tmp_path_factory.mktemp("imagenet"))
    rng = np.random.default_rng(7)
    torch.save(({w: ("class %d" % i,) for i, w in enumerate(WNIDS)}, []), os.path.join(root, "meta.bin"))
    sizes = [(375, 500), (500, 375), (333, 500), (500, 333), (224, 224), (480, 640), (120, 90), (801, 1200), (500, 500),
             (300, 400), (1000, 8)]
    for i, (h, w) in enumerate(sizes):
        d = os.path.join(root, "val", WNIDS[i % 3])
        os.makedirs(d, exist_ok=True)
        img = Image.fromarray(_smooth(h, w, rng))
        if i == 4:
            img = img.convert("L")
        elif i == 5:
            img = img.convert("CMYK")
        img.save(os.path.join(d, "ILSVRC2012_val_%08d.JPEG" % (i + 1)), quality=88)
    torch.manual_seed(0)
    sd = os.path.join(root, "vit_b_random.pth")
    torch.save({k: v.detach().clone() for k, v in vit_base_patch16_224().state_dict().items()}, sd)
    return root, sd


def _read(method_dir):
    ds = perturbation.ImagenetResults(method_dir)
    items = [ds[i] for i in range(len(ds))]
    return {"image": torch.stack([it[0] for it in items]).numpy(), "vis": torch.stack([it[1] for it in items]).numpy(),
            "target": torch.stack([it[2] for it in items]).numpy()}


@pytest.mark.parametrize("vis_class", ["top", "target"])
@pytest.mark.parametrize("method", hdf5_writer.METHODS)
def test_command_equals_cpu_transform_path(tree, tmp_path, method, vis_class):
    import torchvision.transforms as T
    from torchvision.datasets import ImageNet
    data, sd = tree
    root = str(tmp_path / "cmd")
    path = hdf5_writer.main(["--method", method, "--vis-class", vis_class, "--imagenet-validation-path", data,
                             "--batch-size", "4", "--num-workers", "2", "--state-dict", sd, "--root", root])
    args = perturbation.build_parser().parse_args(["--method", method, "--vis-class", vis_class])
    assert path == os.path.join(perturbation.vis_method_dir(args, root), "results.hdf5")

    lrp, orig_lrp, baselines = segmentation.build_generators(method, sd, kind=hdf5_writer.MODEL_KIND[method])
    ds = ImageNet(data, split="val", transform=T.Compose([T.Resize((224, 224)), T.ToTensor()]))
    loader = torch.utils.data.DataLoader(ds, batch_size=4, shuffle=False, num_workers=0)
    ref_dir = str(tmp_path / "ref")
    hdf5_writer.compute_saliency_and_save(loader, ref_dir, method, lrp=lrp, baselines=baselines, orig_lrp=orig_lrp,
                                          vis_class=vis_class)
    got, ref = _read(os.path.dirname(path)), _read(ref_dir)
    assert got["image"].shape == (N_IMAGES, 3, 224, 224) and got["vis"].shape == (N_IMAGES, 1, 224, 224)
    assert np.array_equal(got["target"], [0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2]) and np.array_equal(got["target"], ref["target"])
    for k in ("image", "vis"):
        assert np.array_equal(got[k].view(np.uint32), ref[k].view(np.uint32)), k

    # a rerun replaces the file; the perturbation evaluation reads the directory
    hdf5_writer.main(["--method", method, "--vis-class", vis_class, "--imagenet-validation-path", data,
                      "--batch-size", "5", "--num-workers", "0", "--state-dict", sd, "--root", root])
    again = _read(os.path.dirname(path))
    assert np.array_equal(again["image"].view(np.uint32), got["image"].view(np.uint32))
    res = perturbation.main(["--method", method, "--vis-class", vis_class, "--root", root, "--state-dict", sd,
                             "--batch-size", "4"])
    exp = os.path.join(perturbation.runs_dir(args, root), "experiment_0")
    for name in perturbation.NAMES:
        a = np.load(os.path.join(exp, name + ".npy"))
        assert a.shape[-1] == N_IMAGES and np.array_equal(a, res[name]), name
