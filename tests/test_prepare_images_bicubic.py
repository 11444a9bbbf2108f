"""CPU: the host half of Pillow's bicubic resize (``te_resample_coeffs`` with TE_RESAMPLE_BICUBIC), CLIP's preprocessing.

- The tables against a numpy restatement of Pillow's ``precompute_coeffs`` / ``normalize_coeffs_8bpc`` with the bicubic
  filter (support 2, a = -0.5) for every input size 1..1200 at 224 and for upscaling to odd sizes.
- That restatement, run as the two 8-bit passes with the library's own tables, equals ``PIL.Image.resize(..., BICUBIC)``
  bit for bit, down- and upscaling, odd sizes and an image tall enough for Pillow to resize vertically first: so the
  tables are what the device passes need (the kernels are the bilinear ones, table driven; tests/test_gpu_clip.py runs them).
- The bilinear form of the new entry point is ``te_resize_coeffs``; an unknown filter is refused.
"""
import ctypes

import numpy as np
import pytest
from PIL import Image

from transformer_explainability_b200 import _lib

BICUBIC = _lib.RESAMPLE["bicubic"]


def _cubic(x):
    x = abs(x)
    a = -0.5
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coeffs(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc (Resample.c) with the bicubic filter."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(np.ceil(support)) * 2 + 1
    k = np.zeros((out_size, ksize), np.int32)
    b = np.zeros((out_size, 2), np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_cubic((x + xmin - center + 0.5) / fs) for x in range(xmax)]
        ww = sum(w)
        for x in range(xmax):
            v = w[x] / ww if ww != 0.0 else w[x]
            k[xx, x] = int(-0.5 + v * (1 << 22)) if v < 0 else int(0.5 + v * (1 << 22))
        b[xx] = (xmin, xmax)
    return k, b


def lib_coeffs(in_size, out_size, resample=BICUBIC):
    lib = _lib.load()
    ksize = lib.te_resample_coeffs(in_size, out_size, resample, None, None)
    assert ksize > 0
    k = np.zeros((out_size, ksize), np.int32)
    b = np.zeros((out_size, 2), np.int32)
    assert lib.te_resample_coeffs(in_size, out_size, resample, k.ctypes.data_as(ctypes.c_void_p),
                                  b.ctypes.data_as(ctypes.c_void_p)) == ksize
    return k, b


def _pass(a, k, b, axis):
    """One 8-bit pass of Pillow (int32 sums from 2^21, clip to uint8) along ``axis`` with the tables k, b."""
    a = np.moveaxis(a, axis, 0).astype(np.int64)
    out = np.empty((k.shape[0],) + a.shape[1:], np.uint8)
    for i in range(k.shape[0]):
        lo, n = b[i]
        s = (1 << 21) + np.tensordot(k[i, :n].astype(np.int64), a[lo:lo + n], axes=(0, 0))
        out[i] = np.where(s >= 255 << 22, 255, np.where(s <= 0, 0, s >> 22))
    return np.moveaxis(out, 0, axis)


def resize(a, oh, ow):
    h, w = a.shape[:2]
    if h > w * 100 and oh < h:
        return _pass(_pass(a, *lib_coeffs(h, oh), 0), *lib_coeffs(w, ow), 1)
    return _pass(_pass(a, *lib_coeffs(w, ow), 1), *lib_coeffs(h, oh), 0)


def test_coeffs_match_pillows_precompute():
    for n in range(1, 1201):
        k, b = lib_coeffs(n, 224)
        rk, rb = coeffs(n, 224)
        assert np.array_equal(k, rk) and np.array_equal(b, rb), n
    for n, m in ((7, 224), (13, 61), (224, 227), (1, 5), (301, 299)):
        k, b = lib_coeffs(n, m)
        rk, rb = coeffs(n, m)
        assert np.array_equal(k, rk) and np.array_equal(b, rb), (n, m)


@pytest.mark.parametrize("h,w,oh,ow", [(375, 500, 224, 298), (61, 97, 224, 352), (97, 61, 352, 224), (224, 224, 224, 224),
                                       (5, 3, 17, 11), (299, 301, 223, 225), (1, 1, 3, 3), (1500, 9, 37, 5)])
def test_two_passes_equal_pil_bicubic(h, w, oh, ow):
    rng = np.random.default_rng(h * 7 + w)
    a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    ref = np.asarray(Image.fromarray(a).resize((ow, oh), Image.BICUBIC))
    assert np.array_equal(resize(a, oh, ow), ref)


def test_bilinear_form_and_refusals():
    lib = _lib.load()
    for n, m in ((500, 224), (100, 224), (17, 5)):
        k, b = lib_coeffs(n, m, _lib.RESAMPLE["bilinear"])
        ksize = lib.te_resize_coeffs(n, m, None, None)
        k0, b0 = np.zeros((m, ksize), np.int32), np.zeros((m, 2), np.int32)
        lib.te_resize_coeffs(n, m, k0.ctypes.data_as(ctypes.c_void_p), b0.ctypes.data_as(ctypes.c_void_p))
        assert np.array_equal(k, k0) and np.array_equal(b, b0)
    assert lib.te_resample_coeffs(500, 224, BICUBIC, None, None) == 11
    assert lib.te_resample_coeffs(100, 224, BICUBIC, None, None) == 5
    for bad in (0, 1, 4, -1):
        assert lib.te_resample_coeffs(500, 224, bad, None, None) == -1
        assert lib.te_prepare_images_resample_workspace_bytes(1, 500, 500, 224, 224, bad) == -1
    q = lib.te_prepare_images_resample_workspace_bytes
    assert q(2, 500, 375, 224, 224, _lib.RESAMPLE["bilinear"]) == lib.te_prepare_images_workspace_bytes(2, 500, 375, 224, 224)
    assert q(2, 500, 375, 224, 224, BICUBIC) > q(2, 500, 375, 224, 224, _lib.RESAMPLE["bilinear"])
