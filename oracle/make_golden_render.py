"""Generate ``tests/golden/render.npz`` with cv2: the notebook's own overlay sequence on a few small maps.

    python -m oracle.make_golden_render           # from the repo root, needs cv2

TEST INFRASTRUCTURE.  Stores the JET table of ``cv2.applyColorMap``, and for each of ``MAPS`` (about 64 x 64: peaked,
bimodal, binary, constant-u8, random) the heat map, a seeded image, cv2's Otsu threshold of ``uint8(255 heat)`` and the
overlays of ``Transformer_explainability.ipynb``'s ``generate_visualization`` (``show_cam_on_image`` + ``cvtColor``) with and
without ``use_thresholding``.  ``tests/test_render.py`` checks ``oracle.render`` against it where cv2 is absent.
"""
import os

import numpy as np

H, W = 64, 56
MAPS = ("peaked", "bimodal", "binary", "constant_u8", "random")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "render.npz")


def heat_maps(h=H, w=W, seed=0):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    peaked = np.exp(-((y - 0.3 * h) ** 2 + (x - 0.6 * w) ** 2) / (2 * (0.08 * h) ** 2))
    bimodal = 0.9 * np.exp(-((y - 0.25 * h) ** 2 + (x - 0.25 * w) ** 2) / (2 * (0.1 * h) ** 2)) + \
        0.5 * np.exp(-((y - 0.7 * h) ** 2 + (x - 0.7 * w) ** 2) / (2 * (0.15 * h) ** 2)) + 0.05 * rng.random((h, w))
    binary = (rng.random((h, w)) < 0.3).astype(np.float64)
    constant = np.full((h, w), 0.5)
    rand = rng.random((h, w))
    out = []
    for m in (peaked, bimodal, binary, constant, rand):
        m = m.astype(np.float32)
        if m.max() > m.min():
            m = (m - m.min()) / (m.max() - m.min())
        out.append(m)
    return np.stack(out)


def images(n, h=H, w=W, seed=1):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([x / w, y / h, (x + y) / (h + w)])[None] * 2 - 1
    return (np.round((base + 0.3 * rng.standard_normal((n, 3, h, w))) * 64) / 64).astype(np.float32)   # compresses


def notebook(cv2, image, heat, use_thresholding):
    """``generate_visualization``'s host part on a [3, h, w] image and an [h, w] min-max normalised map."""
    t, ret = heat, None
    if use_thresholding:
        t = (t * 255).astype(np.uint8)
        ret, t = cv2.threshold(t, 0, 255, cv2.THRESH_BINARY + cv2.THRESH_OTSU)
        t[t == 255] = 1
    img = image.transpose(1, 2, 0)
    img = (img - img.min()) / (img.max() - img.min())
    heatmap = cv2.applyColorMap(np.uint8(255 * t), cv2.COLORMAP_JET)
    heatmap = np.float32(heatmap) / 255
    cam = heatmap + np.float32(img)
    cam = cam / np.max(cam)
    vis = np.uint8(255 * cam)
    return cv2.cvtColor(np.array(vis), cv2.COLOR_RGB2BGR), ret


def main():
    import cv2
    heat = heat_maps()
    imgs = images(len(heat))
    jet = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(1, 256), cv2.COLORMAP_JET)[0]
    plain = np.stack([notebook(cv2, i, m, False)[0] for i, m in zip(imgs, heat)])
    thr = [notebook(cv2, i, m, True) for i, m in zip(imgs, heat)]
    np.savez_compressed(OUT, jet_bgr=jet, heat=heat, images=imgs, names=np.array(MAPS),
                        thresholds=np.array([int(r) for _, r in thr], np.int32), overlay=plain,
                        overlay_otsu=np.stack([v for v, _ in thr]), cv2_version=np.array(cv2.__version__))
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
