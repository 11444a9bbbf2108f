"""The notebooks' relevance overlay on the GPU (``te_render_overlay``) against the notebook's per-image cv2 path, and the
overlay command.

    python tools/bench_render.py [--batch 256] [--iters 50] [--images 64] [--command-batch 16]

Reports one JSON line:
* ``kernel`` / ``kernel_otsu``: ``render_overlays`` on a [B, 3, 224, 224] batch already on the device, without and with
  Otsu thresholding (CUDA events over ``--iters`` calls): ms per batch, images/s, and the algorithmic bytes (16 read and
  3 written per pixel) over the time as a share of the H100 SXM's 3.35 TB/s; the output is checked bit for bit against
  ``oracle.render`` on a few samples first;
* ``cpu_cv2`` / ``cpu_cv2_otsu``: the notebook's host sequence (``show_cam_on_image`` + ``cvtColor``, the heat map and the
  image already on the host) per image of the same batch, one host thread, host clock (skipped without cv2);
* ``command``: ``visualization.run`` over ``--images`` synthetic JPEGs of ImageNet-val sizes written to a temporary
  directory, random-init ViT-B/16, centre crop, the predicted class only: images/s after a warm-up run, split into decode,
  GPU (to the end of the device-to-host copy) and PNG encode;
* ``gpu`` / ``power_limit_w``: the card, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import render                                                   # noqa: E402
from transformer_explainability_b200 import _lib, visualization             # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SIZES = [(375, 500), (500, 375), (333, 500), (500, 333), (500, 500)]


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                # noqa: BLE001 — reported as unknown, the measurement itself does not depend on it
        return None


def batch(b, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, 3, 224, 224, generator=g)
    maps = torch.rand(b, 196, generator=g) ** 4
    return x.cuda(), visualization.relevance_to_heatmap(maps.cuda())


def bench_kernel(x, heat, iters, otsu):
    out = visualization.render_overlays(x, heat, otsu)
    xs, hs, got = x[:4].cpu().numpy(), heat[:4].cpu().numpy(), out[:4].cpu().numpy()
    for i in range(4):
        if not np.array_equal(got[i], render.overlay(xs[i], hs[i], otsu)[0]):
            raise SystemExit("te_render_overlay differs from the oracle on sample %d" % i)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        visualization.render_overlays(x, heat, otsu)
    end.record()
    torch.cuda.synchronize()
    s = start.elapsed_time(end) / 1e3 / iters
    nbytes = x.shape[0] * 224 * 224 * (16 + 3)
    return {"ms_per_batch": 1e3 * s, "images_per_s": x.shape[0] / s, "bytes_per_s": nbytes / s,
            "share_of_hbm_peak": nbytes / s / HBM_BYTES_PER_S}


def bench_cpu(x, heat, otsu):
    try:
        import cv2
    except ImportError:
        return None
    from oracle.make_golden_render import notebook
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    cv2.setNumThreads(1)
    xs, hs = x.cpu().numpy(), heat.cpu().numpy()
    t0 = time.perf_counter()
    for i in range(len(xs)):
        notebook(cv2, xs[i], hs[i], otsu)
    s = time.perf_counter() - t0
    torch.set_num_threads(threads)
    return {"ms_per_image": 1e3 * s / len(xs), "images_per_s": len(xs) / s}


def bench_command(n_images, b):
    from PIL import Image
    rng = np.random.default_rng(1)
    with tempfile.TemporaryDirectory(prefix="te_bench_render_") as tmp:
        src = os.path.join(tmp, "in")
        os.makedirs(src)
        for i in range(n_images):
            h, w = SIZES[i % len(SIZES)]
            y, xx = np.mgrid[0:h, 0:w]
            a = np.stack([xx * 255 // (w - 1), y * 255 // (h - 1), (xx + y) * 127 // (h + w - 2)], -1)
            a = a + rng.integers(-30, 31, (h, w, 3))
            Image.fromarray(np.clip(a, 0, 255).astype(np.uint8)).save(os.path.join(src, "img%05d.jpg" % i), quality=90)
        torch.manual_seed(0)
        model = visualization.build_model("vit_base_patch16_224")
        paths = visualization.image_paths([src])
        visualization.run(model, paths[:b], os.path.join(tmp, "warm"), batch_size=b)
        t = {}
        t0 = time.perf_counter()
        visualization.run(model, paths, os.path.join(tmp, "out"), batch_size=b, timings=t)
        total = time.perf_counter() - t0
    return {"images": n_images, "batch": b, "images_per_s": n_images / total,
            "seconds": {k: round(v, 4) for k, v in t.items()}, "total_s": round(total, 4)}


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--images", type=int, default=64)
    p.add_argument("--command-batch", type=int, default=16)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render needs a GPU")
    _lib.load()
    x, heat = batch(args.batch)
    res = {"gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit(), "batch": args.batch,
           "kernel": bench_kernel(x, heat, args.iters, False), "kernel_otsu": bench_kernel(x, heat, args.iters, True),
           "cpu_cv2": bench_cpu(x, heat, False), "cpu_cv2_otsu": bench_cpu(x, heat, True),
           "command": bench_command(args.images, args.command_batch)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
