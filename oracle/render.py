"""Relevance-overlay oracle (TEST INFRASTRUCTURE, numpy only).

Restates the figure of the reference notebooks (``Transformer_explainability.ipynb``: ``generate_visualization`` with
``use_thresholding`` and ``show_cam_on_image``) without cv2, so that it runs where cv2 is absent:

* ``jet_bgr``      the 256-entry uint8 BGR table of ``cv2.applyColorMap(..., COLORMAP_JET)``, derived from JET's piecewise
                   linear definition (see ``te_render.cu``: half-way values to the even neighbour, blue at 159 is 1);
* ``otsu``         OpenCV's ``getThreshVal_Otsu_8u`` loop over the 256-bin histogram, in Python floats (IEEE fp64, no FMA),
                   with its ``FLT_EPSILON`` skips;
* ``overlay``      the whole per-sample sequence, fp32 numpy, returning the uint8 BGR image and the threshold.

``tests/golden/render.npz`` (``make_golden_render``, written with cv2) pins all three.
"""
import numpy as np

FLT_EPSILON = float(np.finfo(np.float32).eps)


def jet_bgr():
    """uint8 [256, 3] BGR: channel c (1 blue, 2 green, 3 red) of level u is clip(1.5 - |4 u / 255 - c|, 0, 1) times 255,
    i.e. k2 / 2 with the integer k2 = clip(765 - 2 |4 u - 255 c|, 0, 510), rounded half to even."""
    u = np.arange(256)[:, None]
    c = np.arange(1, 4)[None, :]
    k2 = np.clip(765 - 2 * np.abs(4 * u - 255 * c), 0, 510)
    lo = k2 // 2
    t = np.where(k2 % 2 == 1, lo + lo % 2, lo)
    t[159, 0] = 1                                  # cv2's fp32 sample of blue at 159 lies below 1.5 / 255
    return t.astype(np.uint8)


def otsu(u8):
    """cv2.threshold(u8, 0, 255, THRESH_BINARY + THRESH_OTSU)[0] as an int."""
    h = np.bincount(np.asarray(u8, np.uint8).reshape(-1), minlength=256).tolist()
    scale = 1.0 / float(sum(h))
    mu = 0.0
    for i in range(256):
        mu += i * float(h[i])
    mu *= scale
    mu1 = q1 = max_sigma = 0.0
    max_val = 0
    for i in range(256):
        p_i = h[i] * scale
        mu1 *= q1
        q1 += p_i
        q2 = 1.0 - q1
        if min(q1, q2) < FLT_EPSILON or max(q1, q2) > 1.0 - FLT_EPSILON:
            continue
        mu1 = (mu1 + i * p_i) / q1
        mu2 = (mu - q1 * mu1) / q2
        sigma = q1 * q2 * (mu1 - mu2) * (mu1 - mu2)
        if sigma > max_sigma:
            max_sigma = sigma
            max_val = i
    return max_val


def to_u8(x):
    """np.uint8 of a float32 array in [0, 256) as numpy casts it on x86-64: truncation, NaN -> 0."""
    x = np.asarray(x, np.float32)
    return np.where(np.isnan(x), 0, np.trunc(np.nan_to_num(x))).astype(np.uint8)


def overlay(image, heat, use_thresholding=False):
    """image [3, h, w] fp32, heat [h, w] fp32 (min-max normalised) -> (uint8 BGR [h, w, 3], Otsu threshold or None)."""
    image = np.asarray(image, np.float32)
    heat = np.asarray(heat, np.float32)
    with np.errstate(all="ignore"):
        u = to_u8(np.float32(255) * heat)
        t = None
        if use_thresholding:
            t = otsu(u)
            u = np.where(u > t, 255, 0).astype(np.uint8)
        img = image.transpose(1, 2, 0)
        img = (img - img.min()) / (img.max() - img.min())
        cam = jet_bgr()[u].astype(np.float32) / np.float32(255) + img
        vis = cam / np.max(cam)
        return to_u8(np.float32(255) * vis)[..., ::-1].copy(), t
