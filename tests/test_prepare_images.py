"""CPU: the input preparation of the generate_visualizations command (``hdf5_writer``) without a device.

``te_resize_coeffs`` (the host half of ``te_prepare_images``) is checked against a numpy restatement of Pillow's
``precompute_coeffs`` + ``normalize_coeffs_8bpc``; the restatement, run as Pillow's two passes, is checked against
``PIL.Image.resize(BILINEAR)`` itself, so Pillow is the pin and no golden file is needed.  Then the workspace query and the
argument checks of ``te_prepare_images``, the command's parser and output directory, the ImageNet reader and the collate.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
from PIL import Image

from transformer_explainability_b200 import _lib, hdf5_writer, perturbation

PRECISION_BITS = 22


# ---- numpy restatement of Pillow's bilinear resize of 8-bit images ------------------------------------------------------
def coeffs(in_size, out_size):
    """(k int64 [out, ksize], bounds int64 [out, 2] = (xmin, n)) of Pillow's precompute_coeffs (bilinear, support 1) and
    normalize_coeffs_8bpc, vectorised over the output index; the weight sum is accumulated in index order as Pillow's."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 1.0 * fs
    ksize = int(np.ceil(support)) * 2 + 1
    center = (np.arange(out_size) + 0.5) * scale
    ss = 1.0 / fs
    xmin = np.maximum(np.trunc(center - support + 0.5).astype(np.int64), 0)
    n = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), in_size) - xmin
    j = np.arange(ksize)
    t = np.abs(((j[None, :] + xmin[:, None]) - center[:, None] + 0.5) * ss)
    w = np.where((j[None, :] < n[:, None]) & (t < 1.0), 1.0 - t, 0.0)
    ww = np.zeros(out_size)
    for c in range(ksize):
        ww = ww + w[:, c]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    scaled = w * (1 << PRECISION_BITS)
    k = np.where(w < 0, np.trunc(-0.5 + scaled), np.trunc(0.5 + scaled)).astype(np.int64)
    return k, np.stack([xmin, n], axis=1)


def resample_axis(a, out_size, axis):
    """One pass over ``axis`` of a uint8 array: int accumulator from 2^21, u8 * k, clip to uint8 (Pillow's clip8)."""
    a = np.moveaxis(a, axis, 0).astype(np.int64)
    k, b = coeffs(a.shape[0], out_size)
    idx = np.minimum(b[:, :1] + np.arange(k.shape[1])[None, :], a.shape[0] - 1)      # weights past n are zero
    s = np.full((out_size,) + a.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for c in range(k.shape[1]):
        s += a[idx[:, c]] * k[:, c].reshape((-1,) + (1,) * (a.ndim - 1))
    out = np.where(s >= 255 << PRECISION_BITS, 255, np.where(s <= 0, 0, s >> PRECISION_BITS)).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(a, oh, ow):
    """Pillow's order: the horizontal pass, its uint8 result, then the vertical pass; Pillow 12's ``Image.resize`` turns
    it round for an image taller than 100 times its width that shrinks vertically."""
    h, w = a.shape[:2]
    if h > w * 100 and oh < h:
        return resample_axis(resample_axis(a, oh, 0), ow, 1)
    return resample_axis(resample_axis(a, ow, 1), oh, 0)


def lib_coeffs(in_size, out_size):
    lib = _lib.load()
    ksize = lib.te_resize_coeffs(in_size, out_size, None, None)
    assert ksize > 0
    k = np.zeros((out_size, ksize), np.int32)
    b = np.zeros((out_size, 2), np.int32)
    assert lib.te_resize_coeffs(in_size, out_size, k.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p)) == ksize
    return k, b


# ---- the tables --------------------------------------------------------------------------------------------------------------
def test_coeffs_every_input_size_at_224():
    for n in range(1, 4097):
        k, b = lib_coeffs(n, 224)
        rk, rb = coeffs(n, 224)
        assert np.array_equal(k, rk) and np.array_equal(b, rb), n


@pytest.mark.parametrize("out_size", [1, 7, 384, 1000])
def test_coeffs_other_outputs(out_size):
    for n in list(range(1, 300)) + list(range(300, 4097, 7)) + [16384]:
        k, b = lib_coeffs(n, out_size)
        rk, rb = coeffs(n, out_size)
        assert np.array_equal(k, rk) and np.array_equal(b, rb), (n, out_size)


SIZES = [(1, 1), (1, 500), (500, 1), (2, 3), (224, 224), (224, 300), (300, 224), (100, 150), (57, 999), (999, 57),
         (375, 500), (500, 375), (500, 333), (333, 500), (500, 500), (1200, 801), (801, 1200), (2000, 3000), (4096, 7),
         (701, 7), (700, 7), (2001, 20), (2000, 20),
         (223, 225), (225, 223), (448, 448), (447, 449), (112, 224), (224, 112), (16, 16), (3000, 224), (77, 1024),
         (1024, 77), (640, 480)]


@pytest.mark.parametrize("hw", SIZES, ids=lambda hw: "%dx%d" % hw)
def test_restatement_equals_pillow(hw):
    h, w = hw
    a = np.random.default_rng(h * 10007 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    ref = np.asarray(Image.fromarray(a).resize((224, 224), Image.BILINEAR))
    assert np.array_equal(resize(a, 224, 224), ref)


def test_restatement_equals_pillow_non_square_outputs():
    a = np.random.default_rng(3).integers(0, 256, (375, 500, 3), dtype=np.uint8)
    for oh, ow in ((100, 384), (384, 100), (1, 7), (7, 1), (1000, 600)):
        ref = np.asarray(Image.fromarray(a).resize((ow, oh), Image.BILINEAR))
        assert np.array_equal(resize(a, oh, ow), ref), (oh, ow)
    a = np.random.default_rng(4).integers(0, 256, (1500, 9, 3), dtype=np.uint8)           # vertical pass first
    for oh, ow in ((224, 224), (1499, 3), (100, 1000), (1500, 20), (2000, 5)):
        ref = np.asarray(Image.fromarray(a).resize((ow, oh), Image.BILINEAR))
        assert np.array_equal(resize(a, oh, ow), ref), (oh, ow)


# ---- workspace query and argument checks -----------------------------------------------------------------------------------
def test_workspace_query():
    lib = _lib.load()
    q = lib.te_prepare_images_workspace_bytes
    a = q(32, 500, 500, 224, 224)
    assert a > 0 and a % 256 == 0
    assert a >= 3 * 32 * 500 * 224                                       # the uint8 intermediate [h, out_w, 3]
    assert q(32, 1000, 500, 224, 224) > a and q(32, 500, 1000, 224, 224) > a and q(64, 500, 500, 224, 224) > a
    for bad in ((0, 500, 500, 224, 224), (65536, 1, 1, 1, 1), (1, 0, 5, 224, 224), (1, 5, 0, 224, 224),
                (1, _lib.PREPARE_MAX_SIDE + 1, 5, 224, 224), (1, 5, _lib.PREPARE_MAX_SIDE + 1, 224, 224),
                (1, 5, 5, 0, 224), (1, 5, 5, 224, _lib.PREPARE_MAX_OUT + 1)):
        assert q(*bad) == -1, bad
    assert q(1, _lib.PREPARE_MAX_SIDE, _lib.PREPARE_MAX_SIDE, _lib.PREPARE_MAX_OUT, _lib.PREPARE_MAX_OUT) > 0


def test_resize_coeffs_errors():
    lib = _lib.load()
    assert lib.te_resize_coeffs(500, 224, None, None) == 7
    assert lib.te_resize_coeffs(100, 224, None, None) == 3
    for bad in ((0, 224), (_lib.PREPARE_MAX_SIDE + 1, 224), (5, 0), (5, _lib.PREPARE_MAX_OUT + 1)):
        assert lib.te_resize_coeffs(*bad, None, None) == -1
    k = np.zeros(224 * 7, np.int32)
    assert lib.te_resize_coeffs(500, 224, k.ctypes.data_as(ctypes.c_void_p), None) == -1
    assert b"both" in lib.te_last_error()


def _call(sizes, offsets, packed_bytes=10 ** 9, batch=None, out_hw=(224, 224), out01=True, out_norm=False, mean=None,
          std=None, ws_bytes=1 << 40):
    """te_prepare_images on fake device addresses: every case here must be refused before anything touches them."""
    lib = _lib.load()
    sz = np.ascontiguousarray(np.asarray(sizes, np.int32).reshape(-1, 2))
    off = np.ascontiguousarray(np.asarray(offsets, np.int64))
    fake = ctypes.c_void_p(1 << 20)
    flt = lambda v: None if v is None else (ctypes.c_float * 3)(*v)      # noqa: E731
    r = lib.te_prepare_images(fake, packed_bytes, len(sz) if batch is None else batch, sz.ctypes.data_as(ctypes.c_void_p),
                              off.ctypes.data_as(ctypes.c_void_p), out_hw[0], out_hw[1], flt(mean), flt(std),
                              fake if out01 else None, fake if out_norm else None, fake, ws_bytes, None)
    return r, lib.te_last_error().decode()


@pytest.mark.parametrize("case,status,msg", [
    (dict(sizes=[[5, 5]], offsets=[0], batch=0), -1, "batch"),
    (dict(sizes=[[5, 5]], offsets=[0], out01=False), -1, "no output"),
    (dict(sizes=[[5, 5]], offsets=[0], out_hw=(0, 224)), -1, "output sides"),
    (dict(sizes=[[5, 5]], offsets=[0], out_hw=(224, 4097)), -1, "output sides"),
    (dict(sizes=[[0, 5]], offsets=[0]), -1, "side"),
    (dict(sizes=[[5, 16385]], offsets=[0]), -1, "side"),
    (dict(sizes=[[5, 5]], offsets=[-1]), -1, "inside the packed buffer"),
    (dict(sizes=[[5, 5], [5, 5]], offsets=[0, 76], packed_bytes=150), -1, "inside the packed buffer"),
    (dict(sizes=[[5, 5]], offsets=[0], out_norm=True), -1, "mean and std"),
    (dict(sizes=[[5, 5]], offsets=[0], out_norm=True, mean=(0.5,) * 3, std=(0.5, 0.0, 0.5)), -1, "non-zero"),
    (dict(sizes=[[5, 5]], offsets=[0], out_norm=True, mean=(float("nan"), 0.5, 0.5), std=(0.5,) * 3), -1, "finite"),
    (dict(sizes=[[500, 375]], offsets=[0], ws_bytes=1024), -2, "workspace too small"),
])
def test_prepare_images_argument_errors(case, status, msg):
    r, err = _call(**case)
    assert r == status and msg in err, (r, err)


def test_prepare_images_accepts_exact_fit_before_the_workspace_check():
    # the last image ends exactly at the end of the buffer: only the (deliberately small) workspace is refused
    r, err = _call(sizes=[[5, 5], [5, 5]], offsets=[0, 75], packed_bytes=150, ws_bytes=0)
    assert r == -2 and "workspace" in err


# ---- the command ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("vis_class", ["top", "target", "index"])
@pytest.mark.parametrize("ablation", [False, True])
@pytest.mark.parametrize("class_id", [0, 243])
def test_output_directory_is_the_perturbation_input(tmp_path, vis_class, ablation, class_id):
    common = ["--method", "lrp_last_layer", "--vis-class", vis_class, "--is-ablation", str(ablation), "--class-id",
              str(class_id)]
    w = hdf5_writer.parse_args(common + ["--imagenet-validation-path", "/nowhere"])
    p = perturbation.build_parser().parse_args(common)
    root = str(tmp_path)
    want = os.path.join(root, "visualizations", "lrp_last_layer",
                        "index_%d" % class_id if vis_class == "index" else
                        os.path.join(vis_class, "ablation" if ablation else "not_ablation"))
    assert perturbation.vis_method_dir(w, root) == perturbation.vis_method_dir(p, root) == want


def test_parser():
    a = hdf5_writer.parse_args(["--method", "attn_gradcam", "--imagenet-validation-path", "x"])
    assert (a.batch_size, a.vis_class, a.class_id, a.is_ablation, a.num_workers, a.lmd) == (1, "top", 0, False, 4, 10)
    assert set(hdf5_writer.METHODS) == set(hdf5_writer.MODEL_KIND)
    assert len(hdf5_writer.METHODS) == 7
    a = hdf5_writer.parse_args(["--method", "full_lrp", "--imagenet-validation-path", "x", "--is-ablation", "True",
                                "--batch-size", "32", "--lmd", "3", "--cls-agn", "--no-ia", "--no-fx", "--no-fgx", "--no-m",
                                "--no-reg", "--num-workers", "0", "--state-dict", "w.pth", "--root", "r"])
    assert a.is_ablation is True and a.batch_size == 32 and a.num_workers == 0 and a.state_dict == "w.pth"
    for bad in ([], ["--imagenet-validation-path", "x"], ["--method", "grad_rollout", "--imagenet-validation-path", "x"],
                ["--method", "lrp"], ["--method", "lrp", "--imagenet-validation-path", "x", "--batch-size", "0"],
                ["--method", "lrp", "--imagenet-validation-path", "x", "--is-ablation", "maybe"]):
        with pytest.raises(SystemExit):
            hdf5_writer.parse_args(bad)


# ---- reader and collate -------------------------------------------------------------------------------------------------------
def make_tree(root, per_class=(2, 3, 1), seed=0):
    """``meta.bin`` + ``val/{wnid}/*.JPEG`` as torchvision's ImageNet expects it; the first file of the second class is
    grayscale.  Returns [(path, target)] in the order ImageNet lists them."""
    rng = np.random.default_rng(seed)
    wnids = ["n01440764", "n01443537", "n01484850"][:len(per_class)]
    torch.save(({w: ("class %d" % i,) for i, w in enumerate(wnids)}, []), os.path.join(root, "meta.bin"))
    out, idx = [], 0
    for c, (w, n) in enumerate(zip(wnids, per_class)):
        os.makedirs(os.path.join(root, "val", w))
        for i in range(n):
            h, wd = int(rng.integers(40, 120)), int(rng.integers(40, 120))
            a = rng.integers(0, 256, (h, wd, 3), dtype=np.uint8)
            img = Image.fromarray(a[..., 0]) if (c == 1 and i == 0) else Image.fromarray(a)
            path = os.path.join(root, "val", w, "ILSVRC2012_val_%08d.JPEG" % (50 - idx))    # names not in class order
            img.save(path, quality=90)
            out.append((path, c))
            idx += 1
    return sorted(out, key=lambda pt: (pt[1], os.path.basename(pt[0])))


def test_reader_order_targets_and_pixels(tmp_path):
    from torchvision.datasets import ImageNet
    expected = make_tree(str(tmp_path))
    ds = ImageNet(str(tmp_path), split="val", loader=hdf5_writer.read_rgb)
    ref = ImageNet(str(tmp_path), split="val")                          # torchvision's own pil_loader
    assert [(p, t) for p, t in ds.samples] == expected
    assert len(ds) == 6
    for i in range(len(ds)):
        a, t = ds[i]
        r, rt = ref[i]
        assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and t == rt == expected[i][1]
        assert np.array_equal(a, np.asarray(r))
    gi = [os.path.basename(p) for p, _ in expected].index("ILSVRC2012_val_00000048.JPEG")      # the grayscale source
    gray = ds[gi][0]                                                    # replicated by convert("RGB")
    assert np.array_equal(gray[..., 0], gray[..., 1]) and np.array_equal(gray[..., 0], gray[..., 2])


def test_collate_packing():
    rng = np.random.default_rng(1)
    samples = [(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), t) for (h, w), t in (((3, 5), 7), ((1, 1), 0),
                                                                                      ((40, 2), 999), ((9, 9), 3))]
    packed, sizes, offsets, targets = hdf5_writer.pack_images(samples)
    assert packed.dtype == torch.uint8 and packed.dim() == 1 and packed.numel() == sum(a.size for a, _ in samples)
    assert sizes.dtype == torch.int32 and sizes.tolist() == [[3, 5], [1, 1], [40, 2], [9, 9]]
    assert offsets.dtype == torch.int64 and offsets.tolist() == [0, 45, 48, 288]
    assert targets.dtype == torch.int64 and targets.tolist() == [7, 0, 999, 3]
    for (a, _), (h, w), o in zip(samples, sizes.tolist(), offsets.tolist()):
        assert np.array_equal(packed[o:o + 3 * h * w].numpy().reshape(h, w, 3), a)
    with pytest.raises(ValueError):
        hdf5_writer.pack_images([(np.zeros((4, 4), np.uint8), 0)])


def test_loader_batches(tmp_path):
    make_tree(str(tmp_path))
    loader = hdf5_writer.imagenet_val_loader(str(tmp_path), batch_size=4, num_workers=0)
    batches = list(loader)
    assert [len(b[3]) for b in batches] == [4, 2]
    assert torch.cat([b[3] for b in batches]).tolist() == [0, 0, 1, 1, 1, 2]
