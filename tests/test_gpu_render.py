"""GPU: ``te_render_overlay`` / ``visualization.render_overlays`` and the overlay command, bit for bit.

* The kernel against ``oracle.render`` fed with the kernel's own ``images`` and ``heat``, with and without Otsu, on seeded
  batches at 224 x 224 and 37 x 61: peaked maps (``relevance_to_heatmap`` of sparse token maps), flat maps, a constant
  relevance map (NaN after min-max), and an image of constant value; the thresholds equal the oracle's.
* A batch equals its samples rendered one at a time.
* Outputs and thresholds pre-filled with 0xFF and 0x5A (as in test_gpu_poison.py) give identical bits, guards intact.
* ``generate_visualization`` equals the previous cv2 path (``show_cam_on_image`` on the same heat map) on a seeded
  ViT-B/16 input, and the notebook's thresholded path, when cv2 imports.
* The command (``visualization.run``) on a small seeded 224 / 16 ViT over PIL-written images of mixed sizes: every PNG equals
  ``generate_visualization(LRP(model), transform(img), class_index)`` of the façade, the centre-crop input equals
  torchvision's transform, ``top_classes.json`` matches the façade's logits, and a batch launches the kernels the module
  docstring states.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import render
from transformer_explainability_b200 import _lib, hdf5_writer, visualization

pytestmark = pytest.mark.gpu


def _batch(h, w, seed):
    """(images [8, 3, h, w], heat [8, h, w]) on the device: samples 0-3 peaked, 4-5 flat, 6 a constant map (NaN), 7 peaked
    on an image of constant value."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(8, 3, h, w, generator=g) * 1.3 + 0.2
    x[7] = 0.37
    maps = torch.rand(8, 196, generator=g) ** 6
    heat = torch.nn.functional.interpolate(maps.reshape(8, 1, 14, 14), size=(h, w), mode="bilinear").reshape(8, h, w)
    lo = heat.reshape(8, -1).amin(1)[:, None, None]
    hi = heat.reshape(8, -1).amax(1)[:, None, None]
    heat = (heat - lo) / (hi - lo)
    heat[4] = torch.rand(h, w, generator=g)
    heat[5] = torch.rand(h, w, generator=g) * 0.5 + 0.25
    if (h, w) == (224, 224):
        maps[6] = 0.25
        heat[:7] = visualization.relevance_to_heatmap(maps[:7].cuda()).cpu()[:7]
        heat[4] = torch.rand(h, w, generator=g)
        heat[5] = torch.rand(h, w, generator=g) * 0.5 + 0.25
    else:
        heat[6] = float("nan")
    assert torch.isnan(heat[6]).all()
    return x.cuda(), heat.cuda()


@pytest.mark.parametrize("otsu", [False, True])
@pytest.mark.parametrize("hw", [(224, 224), (37, 61)], ids=lambda hw: "%dx%d" % hw)
def test_kernel_equals_oracle(hw, otsu):
    for seed in (0, 1):
        x, heat = _batch(*hw, seed)
        out, thr = visualization.render_overlays(x, heat, use_thresholding=otsu, return_thresholds=True)
        assert out.shape == (8, hw[0], hw[1], 3) and out.dtype == torch.uint8
        xs, hs, got = x.cpu().numpy(), heat.cpu().numpy(), out.cpu().numpy()
        for i in range(8):
            want, t = render.overlay(xs[i], hs[i], use_thresholding=otsu)
            assert np.array_equal(got[i], want), (seed, i, int((got[i] != want).sum()))
            if otsu:
                assert int(thr[i]) == t, (seed, i)
        assert thr is None if not otsu else thr.dtype == torch.int32
        assert not got[7].any()                                    # constant image: every cam is NaN
        assert got[0].any()


@pytest.mark.parametrize("otsu", [False, True])
def test_batch_equals_samples_alone(otsu):
    x, heat = _batch(224, 224, 2)
    out, thr = visualization.render_overlays(x, heat, use_thresholding=otsu, return_thresholds=True)
    for i in range(8):
        o, t = visualization.render_overlays(x[i:i + 1], heat[i:i + 1], use_thresholding=otsu, return_thresholds=True)
        assert torch.equal(o[0], out[i]), i
        if otsu:
            assert torch.equal(t[0], thr[i])


GUARD = 1 << 16


@pytest.mark.parametrize("otsu", [0, 1])
def test_poisoned_outputs(otsu):
    x, heat = _batch(224, 224, 3)
    lib = _lib.load()
    n = 8 * 224 * 224 * 3
    base = None
    for pattern in (0xFF, 0x5A):
        out = torch.full((n + GUARD,), pattern, dtype=torch.uint8, device="cuda")
        thr = torch.full((8 * 4 + GUARD,), pattern, dtype=torch.uint8, device="cuda")
        r = lib.te_render_overlay(_lib.ptr(x), _lib.ptr(heat), 8, 224, 224, otsu, _lib.ptr(out), _lib.ptr(thr),
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert r == 0, lib.te_last_error()
        torch.cuda.synchronize()
        got = (out[:n].clone(), thr[:32].clone())
        assert bool((out[n:] == pattern).all()) and bool((thr[32:] == pattern).all())
        if not otsu:
            assert bool((got[1] == pattern).all())               # thresholds are only written when thresholding
        if base is None:
            base = got
        else:
            assert torch.equal(got[0], base[0])
            if otsu:
                assert torch.equal(got[1], base[1])
    assert torch.equal(base[0].reshape(8, 224, 224, 3), visualization.render_overlays(x, heat, bool(otsu)))


def test_generate_visualization_equals_cv2_path():
    cv2 = pytest.importorskip("cv2")
    from oracle import vit as ovit
    from oracle.make_golden_render import notebook
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import VisionTransformer
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    params, _ = ovit.init_params("vit_base_patch16_224", seed=0)
    m = VisionTransformer(patch_size=16, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True)
    m.load_state_dict(params)
    m = m.cuda().eval()
    img = torch.randn(3, 224, 224, generator=torch.Generator().manual_seed(1))
    gen = LRP(m)
    for class_index in (None, 7):
        maps = gen.generate_LRP(img.unsqueeze(0).cuda(), method="transformer_attribution", index=class_index).detach()
        heat = visualization.relevance_to_heatmap(maps)[0].cpu().numpy()
        # the previous implementation of generate_visualization, line for line
        im = img.permute(1, 2, 0).numpy()
        im = (im - im.min()) / (im.max() - im.min())
        old = cv2.cvtColor(np.array(np.uint8(255 * visualization.show_cam_on_image(im, heat))), cv2.COLOR_RGB2BGR)
        got = visualization.generate_visualization(gen, img, class_index)
        assert got.dtype == np.uint8 and np.array_equal(got, old), class_index
        want, _ = notebook(cv2, img.numpy(), heat, True)
        assert np.array_equal(visualization.generate_visualization(gen, img, class_index, use_thresholding=True), want)
    batch = torch.stack([img, img.flip(1)])
    many = visualization.generate_visualizations(gen, batch).cpu().numpy()
    assert np.array_equal(many[0], visualization.generate_visualization(gen, img))


# ---- the command end to end ------------------------------------------------------------------------------------------------
IMAGE_SIZES = [(300, 400), (256, 256), (480, 256), (256, 700), (120, 90), (333, 500), (300, 400), (500, 333)]


@pytest.fixture(scope="module")
def small_model():
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import VisionTransformer
    torch.manual_seed(0)
    m = VisionTransformer(img_size=224, patch_size=16, embed_dim=64, depth=2, num_heads=4, mlp_ratio=4, qkv_bias=True,
                          num_classes=10)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    d = tmp_path_factory.mktemp("photos")
    rng = np.random.default_rng(5)
    for i, (h, w) in enumerate(IMAGE_SIZES):
        y, x = np.mgrid[0:h, 0:w]
        a = np.stack([x * 255 // w, y * 255 // h, (x + y) * 127 // (h + w)], -1) + rng.integers(-30, 31, (h, w, 3))
        Image.fromarray(np.clip(a, 0, 255).astype(np.uint8)).save(str(d / ("img%02d.%s" % (i, "png" if i % 2 else "jpg"))))
    return str(d)


def _transform(name):
    import torchvision.transforms as T
    norm = T.Normalize(mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5])
    if name == "resize":
        return T.Compose([T.Resize((224, 224)), T.ToTensor(), norm])
    return T.Compose([T.Resize(256), T.CenterCrop(224), T.ToTensor(), norm])


@pytest.mark.parametrize("transform", ["center-crop", "resize"])
def test_prepared_input_equals_torchvision(folder, transform):
    paths = visualization.image_paths([folder])
    packed, sizes, offsets, _ = hdf5_writer.pack_images([(hdf5_writer.read_rgb(p), 0) for p in paths])
    x, calls = visualization.prepare_batch(packed.cuda(), sizes.numpy(), offsets.numpy(), transform)
    t = _transform(transform)
    ref = torch.stack([t(Image.fromarray(hdf5_writer.read_rgb(p))) for p in paths])
    assert torch.equal(x.cpu(), ref)
    assert calls == (1 if transform == "resize" else len({visualization.center_crop_geometry(h, w)[0]
                                                          for h, w in sizes.tolist()}))


@pytest.mark.parametrize("transform,otsu", [("center-crop", False), ("resize", True)])
def test_command_equals_facade(small_model, folder, tmp_path, transform, otsu):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    out = str(tmp_path / "figs")
    paths = visualization.image_paths([folder])
    written = visualization.run(small_model, paths, out, class_indices=(3, 7), use_thresholding=otsu, transform=transform,
                                batch_size=5)
    top = json.load(open(os.path.join(out, "top_classes.json")))
    assert len(written) == 3 * len(paths) and len(top) == len(paths)
    t = _transform(transform)
    gen = LRP(small_model)
    for p in paths:
        stem = os.path.splitext(os.path.basename(p))[0]
        x = t(Image.fromarray(hdf5_writer.read_rgb(p)))
        logits = small_model(x.unsqueeze(0).cuda())[0].cpu()
        pred = int(logits.argmax())
        want_top = logits.topk(5)[1].tolist()
        assert top[stem]["predicted"] == pred and [e["index"] for e in top[stem]["top5"]] == want_top
        assert [e["logit"] for e in top[stem]["top5"]] == [float(np.float32(logits[i])) for i in want_top]
        probs = torch.softmax(logits[None], dim=1)[0]
        assert np.allclose([e["prob"] for e in top[stem]["top5"]], [float(probs[i]) for i in want_top], rtol=1e-6, atol=0)
        for c in (None, 3, 7):
            png = os.path.join(out, "%s_%d.png" % (stem, pred if c is None else c))
            want = visualization.generate_visualization(gen, x, c, use_thresholding=otsu)
            assert np.array_equal(np.asarray(Image.open(png)), want), (png, c)


def test_launches_per_batch(small_model, folder):
    lib = _lib.load()
    paths = visualization.image_paths([folder])[:5]
    packed, sizes, offsets, _ = hdf5_writer.pack_images([(hdf5_writer.read_rgb(p), 0) for p in paths])
    packed = packed.cuda()
    x, groups = visualization.prepare_batch(packed, sizes.numpy(), offsets.numpy(), "center-crop")
    eng = small_model.engine()
    c0 = lib.te_kernel_launch_count()
    eng.forward(x)
    c1 = lib.te_kernel_launch_count()
    eng.attribute(index=torch.zeros(len(paths), dtype=torch.int32, device="cuda"))
    c2 = lib.te_kernel_launch_count()
    f, a = c1 - c0, c2 - c1
    for transform, g in (("center-crop", groups), ("resize", 1)):
        for classes in ((), (3, 7)):
            before = lib.te_kernel_launch_count()
            visualization.render_batch(small_model, packed, sizes.numpy(), offsets.numpy(), transform, classes)
            k = 1 + len(classes)
            assert lib.te_kernel_launch_count() - before == 2 * g + f + k * (a + 2), (transform, classes)
    assert groups >= 2
