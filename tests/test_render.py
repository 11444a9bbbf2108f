"""CPU: the overlay of the notebooks (``oracle.render``, ``te_render_overlay``'s argument checks) and the overlay command's host
side, without a device.

The oracle's JET table, Otsu thresholds and overlays are pinned to ``tests/golden/render.npz`` (written with cv2 by
``oracle/make_golden_render.py``) and, where cv2 imports, to cv2 itself: all 256 JET entries, Otsu on 200 seeded maps
of several shapes, and the notebook's ``show_cam_on_image`` sequence.  The centre-crop rule of the command is checked
against torchvision's ``Resize(256) + CenterCrop(224)`` on PIL images.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import render
from oracle.make_golden_render import notebook
from transformer_explainability_b200 import _lib, visualization

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "render.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_jet_table_matches_golden(golden):
    assert golden["jet_bgr"].shape == (256, 3)
    assert np.array_equal(render.jet_bgr(), golden["jet_bgr"])


def test_otsu_and_overlays_match_golden(golden):
    assert list(golden["names"]) == ["peaked", "bimodal", "binary", "constant_u8", "random"]
    for i, name in enumerate(golden["names"]):
        plain, t0 = render.overlay(golden["images"][i], golden["heat"][i])
        otsu, t = render.overlay(golden["images"][i], golden["heat"][i], use_thresholding=True)
        assert t0 is None
        assert t == golden["thresholds"][i], name
        assert np.array_equal(plain, golden["overlay"][i]), name
        assert np.array_equal(otsu, golden["overlay_otsu"][i]), name


def test_jet_table_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    ref = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(1, 256), cv2.COLORMAP_JET)[0]
    assert np.array_equal(render.jet_bgr(), ref)


def _maps(rng, n):
    """Seeded u8 maps: uniform, peaked, bimodal, sparse, binary, constant, two-level, of several shapes."""
    out = []
    for i in range(n):
        h, w = [(224, 224), (64, 56), (1, 7), (31, 300)][i % 4]
        kind = i % 7
        if kind == 0:
            a = rng.integers(0, 256, (h, w))
        elif kind == 1:
            a = 255 * np.exp(-rng.random((h, w)) * 8)
        elif kind == 2:
            a = np.where(rng.random((h, w)) < 0.4, rng.normal(60, 15, (h, w)), rng.normal(190, 20, (h, w)))
        elif kind == 3:
            a = np.where(rng.random((h, w)) < 0.02, 255, rng.integers(0, 3, (h, w)))
        elif kind == 4:
            a = np.where(rng.random((h, w)) < 0.5, 0, 255)
        elif kind == 5:
            a = np.full((h, w), rng.integers(0, 256))
        else:
            a = np.where(rng.random((h, w)) < 0.001, 200, 17)
        out.append(np.clip(a, 0, 255).astype(np.uint8))
    return out


def test_otsu_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    for i, u in enumerate(_maps(np.random.default_rng(0), 200)):
        ret, _ = cv2.threshold(u, 0, 255, cv2.THRESH_BINARY + cv2.THRESH_OTSU)
        assert render.otsu(u) == int(ret), i


def test_overlay_matches_notebook_with_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    for i in range(12):
        h, w = [(224, 224), (40, 72)][i % 2]
        heat = rng.random((h, w)).astype(np.float32) ** (1 + i % 4)
        heat = (heat - heat.min()) / (heat.max() - heat.min())
        img = rng.standard_normal((3, h, w)).astype(np.float32) * (1 + i)
        for thr in (False, True):
            want, ret = notebook(cv2, img, heat, thr)
            got, t = render.overlay(img, heat, use_thresholding=thr)
            assert np.array_equal(got, want), (i, thr)
            assert t == (int(ret) if thr else None)


def test_overlay_nan_rules():
    """A NaN heat map (constant relevance) renders as level 0; a constant image makes every sample value 0."""
    img = np.random.default_rng(2).standard_normal((3, 8, 9)).astype(np.float32)
    nan = np.full((8, 9), np.nan, np.float32)
    zero = np.zeros((8, 9), np.float32)
    assert np.array_equal(render.overlay(img, nan)[0], render.overlay(img, zero)[0])
    assert render.overlay(img, nan, True)[1] == 0
    flat, _ = render.overlay(np.full((3, 8, 9), 0.25, np.float32), np.random.default_rng(3).random((8, 9)))
    assert not flat.any()


# ---- render_overlays / te_render_overlay refuse bad input -------------------------------------------------------------------
def test_render_overlays_rejects_cpu_and_misshaped_input():
    x, h = torch.zeros(2, 3, 8, 9), torch.zeros(2, 8, 9)
    with pytest.raises(ValueError, match="CUDA"):
        visualization.render_overlays(x, h)
    for bad_x, bad_h in ((torch.zeros(2, 4, 8, 9), h), (torch.zeros(3, 8, 9), h), (x, torch.zeros(3, 8, 9)),
                         (x, torch.zeros(2, 9, 8)), (x, torch.zeros(2, 8, 9, 1)), (torch.zeros(0, 3, 8, 9), torch.zeros(0, 8, 9)),
                         (torch.zeros(1, 3, 0, 9), torch.zeros(1, 0, 9))):
        with pytest.raises(ValueError, match="expected"):
            visualization.render_overlays(bad_x, bad_h)


@pytest.mark.parametrize("case,msg", [
    (dict(batch=0), "batch"),
    (dict(batch=-3), "batch"),
    (dict(h=0), "h and w"),
    (dict(w=-1), "h and w"),
    (dict(h=40000, w=40000), "int32"),
    (dict(otsu=2), "otsu"),
    (dict(otsu=-1), "otsu"),
    (dict(images=None), "null"),
    (dict(heat=None), "null"),
    (dict(out=None), "null"),
])
def test_render_overlay_argument_errors(case, msg):
    """Every case is refused before anything touches the (fake) device addresses, and nothing is launched."""
    lib = _lib.load()
    fake = ctypes.c_void_p(1 << 20)
    a = dict(images=fake, heat=fake, batch=2, h=8, w=9, otsu=1, out=fake)
    a.update(case)
    before = lib.te_kernel_launch_count()
    r = lib.te_render_overlay(a["images"], a["heat"], a["batch"], a["h"], a["w"], a["otsu"], a["out"], fake, None)
    assert r == -1 and msg in lib.te_last_error().decode(), (r, lib.te_last_error())
    assert lib.te_kernel_launch_count() == before


# ---- the command's host side --------------------------------------------------------------------------------------------------
def test_parser():
    a = visualization.parse_args(["--images", "a.jpg", "d", "--output-dir", "o"])
    assert (a.images, a.output_dir, a.model, a.state_dict, a.class_index, a.use_thresholding, a.transform, a.batch_size) == \
        (["a.jpg", "d"], "o", "vit_base_patch16_224", None, [], False, "center-crop", 16)
    assert visualization.parse_args(["--images", "x", "--output-dir", "o", "--model", "deit_base_patch16_224"]).transform == "resize"
    assert visualization.parse_args(["--images", "x", "--output-dir", "o", "--model", "deit_base_patch16_224",
                                     "--transform", "center-crop"]).transform == "center-crop"
    a = visualization.parse_args(["--images", "x", "--output-dir", "o", "--model", "vit_large_patch16_224", "--class-index",
                                  "243", "282", "--use-thresholding", "--transform", "resize", "--batch-size", "3",
                                  "--state-dict", "w.pth"])
    assert (a.class_index, a.use_thresholding, a.transform, a.batch_size, a.state_dict) == ([243, 282], True, "resize", 3, "w.pth")
    for bad in ([], ["--images", "x"], ["--output-dir", "o"], ["--images", "x", "--output-dir", "o", "--batch-size", "0"],
                ["--images", "x", "--output-dir", "o", "--model", "vit_tiny"],
                ["--images", "x", "--output-dir", "o", "--transform", "crop"]):
        with pytest.raises(SystemExit):
            visualization.parse_args(bad)


CROP_SIZES = [(256, 256), (256, 300), (300, 256), (256, 257), (375, 500), (500, 375), (333, 500), (500, 333), (224, 224),
              (100, 150), (150, 100), (257, 256), (480, 640), (1200, 801), (37, 1000), (1000, 37), (255, 511), (301, 256)]


@pytest.mark.parametrize("hw", CROP_SIZES, ids=lambda hw: "%dx%d" % hw)
def test_center_crop_rule_equals_torchvision(hw):
    import torchvision.transforms as T
    h, w = hw
    img = Image.fromarray(np.random.default_rng(h * 7919 + w).integers(0, 256, (h, w, 3), dtype=np.uint8))
    (rh, rw), (top, left) = visualization.center_crop_geometry(h, w)
    resized = T.Resize(256)(img)
    assert resized.size == (rw, rh)
    assert min(rh, rw) == 256 and 0 <= top <= rh - 224 and 0 <= left <= rw - 224
    assert np.array_equal(np.asarray(resized)[top:top + 224, left:left + 224], np.asarray(T.CenterCrop(224)(resized)))


def test_image_paths_and_output_layout(tmp_path):
    d = tmp_path / "in"
    d.mkdir()
    for name in ("b.png", "a.JPEG", "c.bmp"):
        Image.new("RGB", (5, 4)).save(str(d / name))
    (d / "notes.txt").write_text("not an image")
    (d / "sub").mkdir()
    extra = tmp_path / "z.jpg"
    Image.new("RGB", (3, 3)).save(str(extra))
    got = visualization.image_paths([str(d), str(extra)])
    assert got == [str(d / "a.JPEG"), str(d / "b.png"), str(d / "c.bmp"), str(extra)]
    Image.new("RGB", (3, 3)).save(str(tmp_path / "a.png"))
    with pytest.raises(ValueError, match="stem"):
        visualization.image_paths([str(d), str(tmp_path / "a.png")])
    with pytest.raises(FileNotFoundError):
        visualization.image_paths([str(tmp_path / "missing.jpg")])
