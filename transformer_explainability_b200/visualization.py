"""``generate_visualization`` of the reference notebooks (``example.ipynb:55-66``, ``Transformer_explainability.ipynb``),
batched on the GPU, and the command that renders a folder of images the way the notebooks render one.

relevance [B,196] -> reshape 14x14 -> bilinear x16 (align_corners=False) -> per-sample min-max -> [B,224,224]
(``relevance_to_heatmap``, ``te_relevance_heatmap``), then the JET overlay -> uint8 [B,224,224,3] (``render_overlays``,
``te_render_overlay``): the notebook's numpy / cv2 sequence bit for bit, including the Otsu thresholding of
``use_thresholding``.  Nothing of the figure runs on the host; ``show_cam_on_image`` is kept as the reference-named cv2
function.

    python -m transformer_explainability_b200.visualization --images photos/ --output-dir figures/ \\
        --state-dict vit_base_patch16_224.pth --class-index 243 282

writes ``figures/{stem}_{class}.png`` for the predicted class and every ``--class-index`` of each image, and
``figures/top_classes.json`` (``print_top_classes``' top-5 indices, logits and probabilities per image).  The images are
decoded by PIL on the host and resized on the GPU (``ops.prepare_images``).  ``--transform center-crop`` is
``Resize(256) + CenterCrop(224)`` of ``example.ipynb`` (the default for the ViT models), ``resize`` is ``Resize((224, 224))``
of ``DeiT_example.ipynb`` (the default for DeiT).  Per batch of B images and K classes (the predicted one plus the
``--class-index`` values), the library launches 2 G + F + K (A + 2) kernels (``te_kernel_launch_count``): G
``te_prepare_images`` calls of two launches, one per distinct resized size (G = 1 for ``resize``), the F launches of one
engine forward, and per class the A launches of one ``attribute`` on that same forward, one ``te_relevance_heatmap`` and one
``te_render_overlay``; then one device-to-host copy carries the overlays and the top-5 table.
"""
import argparse
import json
import os
import time

import numpy as np
import torch

from ._host import to_host

MODELS = ("vit_base_patch16_224", "vit_large_patch16_224", "deit_base_patch16_224")
MEAN = STD = (0.5, 0.5, 0.5)            # transforms.Normalize of the notebooks


def relevance_to_heatmap(maps, grid=14, scale=16):
    """[B, grid*grid] -> min-max normalised [B, grid*scale, grid*scale] (device tensor) through the engine's kernel
    (``te_relevance_heatmap``, one block per sample).  CUDA tensors only: there is no host path."""
    if not maps.is_cuda:
        raise ValueError("relevance_to_heatmap needs a CUDA tensor (no CPU fallback)")
    if maps.dim() != 2 or maps.shape[1] != grid * grid:
        raise ValueError("relevance_to_heatmap: maps %s, expected [B, grid*grid] = [B, %d]" % (tuple(maps.shape), grid * grid))
    b = maps.shape[0]
    from . import _lib
    m = maps.detach().to(torch.float32).contiguous()
    out = torch.empty(b, grid * scale, grid * scale, device=m.device, dtype=torch.float32)
    with torch.cuda.device(m.device):
        _lib.check(_lib.load().te_relevance_heatmap(_lib.ptr(m), b, grid, scale, _lib.ptr(out),
                                                    _lib.ctypes.c_void_p(torch.cuda.current_stream(m.device).cuda_stream)),
                   "te_relevance_heatmap")
    return out


def render_overlays(images, heat, use_thresholding=False, return_thresholds=False):
    """The notebook's overlay of ``heat`` [B, h, w] (min-max normalised) on ``images`` [B, 3, h, w] (the normalised model
    input) -> uint8 CUDA [B, h, w, 3], bit for bit ``generate_visualization``'s numpy / cv2 result (``te_render_overlay``).
    ``use_thresholding``: Otsu-threshold ``uint8(255 heat)`` first, as ``Transformer_explainability.ipynb`` does;
    ``return_thresholds`` also returns the int32 CUDA [B] thresholds (None without thresholding).  CUDA tensors only."""
    if images.dim() != 4 or images.shape[1] != 3 or heat.dim() != 3 or heat.shape[0] != images.shape[0] or \
            tuple(heat.shape[1:]) != tuple(images.shape[2:]) or images.numel() == 0:
        raise ValueError("render_overlays: images %s and heat %s, expected [B, 3, h, w] and [B, h, w] with B, h, w >= 1"
                         % (tuple(images.shape), tuple(heat.shape)))
    if not (images.is_cuda and heat.is_cuda):
        raise ValueError("render_overlays needs CUDA tensors (no CPU fallback)")
    if images.device != heat.device:
        raise ValueError("render_overlays: images and heat must be on the same device")
    from . import _lib
    b, _, h, w = images.shape
    x = images.detach().to(torch.float32).contiguous()
    m = heat.detach().to(torch.float32).contiguous()
    out = torch.empty(b, h, w, 3, device=x.device, dtype=torch.uint8)
    thr = torch.empty(b, device=x.device, dtype=torch.int32) if use_thresholding else None
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().te_render_overlay(_lib.ptr(x), _lib.ptr(m), b, h, w, int(bool(use_thresholding)),
                                                 _lib.ptr(out), _lib.ptr(thr),
                                                 _lib.ctypes.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)),
                   "te_render_overlay")
    return (out, thr) if return_thresholds else out


def show_cam_on_image(img, mask):
    """``example.ipynb:48-53``: JET heat-map overlay (host, needs cv2)."""
    import cv2
    heatmap = cv2.applyColorMap(np.uint8(255 * mask), cv2.COLORMAP_JET)
    heatmap = np.float32(heatmap) / 255
    cam = heatmap + np.float32(img)
    return cam / np.max(cam)


# transformer_attribution (the notebooks' method) or the LRP-free gradient-weighted attention rollout of the authors'
# follow-up paper (Chefer, Gur, Wolf, ICCV 2021)
METHODS = ("transformer_attribution", "attn_grad_rollout")


def _check_method(method):
    if method not in METHODS:
        raise ValueError("unknown visualization method %r (expected one of %s)" % (method, ", ".join(METHODS)))


def generate_visualization(attribution_generator, original_image, class_index=None, start_layer=0, use_thresholding=False,
                           method="transformer_attribution"):
    """``example.ipynb:55-66`` / ``Transformer_explainability.ipynb``: original_image [3,224,224] -> uint8 overlay
    [224,224,3] (numpy), with the notebook's ``use_thresholding`` switch; ``method`` one of ``METHODS``."""
    _check_method(method)
    dev = next(attribution_generator.model.parameters()).device
    x = original_image.unsqueeze(0).to(dev)
    if method == "attn_grad_rollout":
        maps = attribution_generator.generate_attn_grad_rollout(x, index=class_index, start_layer=start_layer)
    else:
        maps = attribution_generator.generate_LRP(x, method="transformer_attribution", index=class_index,
                                                  start_layer=start_layer).detach()
    return render_overlays(x, relevance_to_heatmap(maps), use_thresholding)[0].cpu().numpy()


def generate_visualizations(attribution_generator, images, class_index=None, start_layer=0, use_thresholding=False,
                            method="transformer_attribution"):
    """``generate_visualization`` for a batch: images [B,3,224,224] -> uint8 CUDA [B,224,224,3].  One engine call
    (``generate_LRP_batched`` or ``generate_attn_grad_rollout``) for the maps, one ``te_relevance_heatmap`` and one
    ``te_render_overlay``."""
    _check_method(method)
    dev = next(attribution_generator.model.parameters()).device
    x = images.to(dev, torch.float32)
    if method == "attn_grad_rollout":
        maps = attribution_generator.generate_attn_grad_rollout(x, index=class_index, start_layer=start_layer)
    else:
        maps = attribution_generator.generate_LRP_batched(x, index=class_index, start_layer=start_layer)
    return render_overlays(x, relevance_to_heatmap(maps), use_thresholding)


# ---- the command -------------------------------------------------------------------------------------------------------------
def center_crop_geometry(h, w, size=256, crop=224):
    """torchvision's ``Resize(size)`` + ``CenterCrop(crop)`` on an h x w PIL image: ((resized h, resized w), (top, left)).
    The short side becomes ``size``, the long side ``int(size * long / short)``; the offsets are
    ``int(round((s - crop) / 2))``."""
    if w <= h:
        rh, rw = int(size * h / w), size
    else:
        rh, rw = size, int(size * w / h)
    return (rh, rw), (int(round((rh - crop) / 2.0)), int(round((rw - crop) / 2.0)))


def prepare_batch(packed, sizes, offsets, transform, size=224):
    """Normalised model input [B, 3, size, size] of a packed batch (``hdf5_writer.pack_images``, packed on the device):
    ``resize`` is one ``ops.prepare_images`` call; ``center-crop`` is one call per distinct resized size, each cropped by a
    view.  Returns (images, number of ``prepare_images`` calls)."""
    from . import ops
    sizes = np.asarray(sizes).reshape(-1, 2)
    offsets = np.asarray(offsets).reshape(-1)
    if transform == "resize":
        _, x = ops.prepare_images(packed, sizes, offsets, (size, size), mean=MEAN, std=STD)
        return x, 1
    geo = [center_crop_geometry(int(h), int(w), crop=size) for h, w in sizes]
    x = torch.empty(len(sizes), 3, size, size, device=packed.device, dtype=torch.float32)
    groups = {}
    for i, (rs, _) in enumerate(geo):
        groups.setdefault(rs, []).append(i)
    for (rh, rw), idx in groups.items():
        _, y = ops.prepare_images(packed, sizes[idx], offsets[idx], (rh, rw), mean=MEAN, std=STD)
        for j, i in enumerate(idx):
            top, left = geo[i][1]
            x[i] = y[j, :, top:top + size, left:left + size]
    return x, len(groups)


def image_paths(inputs):
    """Files named on the command line, and the image files (by PIL's registered extensions) of each directory, sorted."""
    from PIL import Image
    exts = {e.lower() for e in Image.registered_extensions()}
    out = []
    for p in inputs:
        if os.path.isdir(p):
            out.extend(sorted(os.path.join(p, f) for f in os.listdir(p)
                              if os.path.splitext(f)[1].lower() in exts and os.path.isfile(os.path.join(p, f))))
        elif os.path.isfile(p):
            out.append(p)
        else:
            raise FileNotFoundError(p)
    stems = [os.path.splitext(os.path.basename(p))[0] for p in out]
    dup = sorted({s for s in stems if stems.count(s) > 1})
    if dup:
        raise ValueError("two inputs share the file stem %r: their overlays would overwrite each other" % dup[0])
    return out


def build_model(name, state_dict=None, device="cuda"):
    """The ``ViT_LRP`` model of the notebooks, with weights of timm key names from ``state_dict`` (nothing is downloaded)."""
    from .baselines.ViT import ViT_LRP
    model = getattr(ViT_LRP, name)()
    if state_dict:
        model.load_state_dict(torch.load(state_dict, map_location="cpu"))
    return model.to(device).eval()


def render_batch(model, packed, sizes, offsets, transform, class_indices=(), use_thresholding=False,
                 method="transformer_attribution"):
    """One batch of the command on the device: (overlays uint8 [B, K, 224, 224, 3], classes int64 [B, K], top-5 indices
    [B, k], logits [B, k], probabilities [B, k]) on the host after one device-to-host copy; K = 1 + len(class_indices),
    column 0 the predicted class.  ``method``: one of ``METHODS``."""
    from . import _lib
    _check_method(method)
    x, _ = prepare_batch(packed, sizes, offsets, transform)
    eng = model.engine()
    flags = eng.flags | (_lib.FLAG_ATTN_GRAD_ROLLOUT if method == "attn_grad_rollout" else 0)
    logits = eng.forward(x)
    b = x.shape[0]
    pred = logits.argmax(dim=-1)
    cols = [pred] + [torch.full((b,), int(c), device=pred.device, dtype=pred.dtype) for c in class_indices]
    overlays = []
    for idx in cols:
        maps, _ = eng.attribute(index=idx.to(torch.int32), flags=flags)
        overlays.append(render_overlays(x, relevance_to_heatmap(maps), use_thresholding))
    top = logits.topk(min(5, logits.shape[1]), dim=1)[1]
    return to_host(torch.stack(overlays, 1), torch.stack(cols, 1), top, logits.gather(1, top),
                   torch.softmax(logits, dim=1).gather(1, top))


def run(model, paths, output_dir, class_indices=(), use_thresholding=False, transform="center-crop", batch_size=16,
        timings=None, method="transformer_attribution"):
    """The command on already-parsed arguments; returns the written PNG paths.  ``timings`` (a dict) accumulates the
    seconds spent decoding, on the device (ending in the copy to the host) and encoding PNGs."""
    from PIL import Image
    from . import hdf5_writer
    os.makedirs(output_dir, exist_ok=True)
    t = timings if timings is not None else {}
    for key in ("decode", "gpu", "encode"):
        t.setdefault(key, 0.0)
    written, top = [], {}
    dev = next(model.parameters()).device
    for s in range(0, len(paths), batch_size):
        chunk = paths[s:s + batch_size]
        t0 = time.perf_counter()
        packed, sizes, offsets, _ = hdf5_writer.pack_images([(hdf5_writer.read_rgb(p), 0) for p in chunk])
        t1 = time.perf_counter()
        img, cls, idx, logit, prob = render_batch(model, packed.to(dev), sizes.numpy(), offsets.numpy(), transform,
                                                  class_indices, use_thresholding, method)
        t2 = time.perf_counter()
        for i, p in enumerate(chunk):
            stem = os.path.splitext(os.path.basename(p))[0]
            for j in range(cls.shape[1]):
                out = os.path.join(output_dir, "%s_%d.png" % (stem, int(cls[i, j])))
                Image.fromarray(img[i, j]).save(out)
                written.append(out)
            top[stem] = {"file": os.path.abspath(p), "predicted": int(cls[i, 0]),
                         "top5": [{"index": int(a), "logit": float(b), "prob": float(c)}
                                  for a, b, c in zip(idx[i], logit[i], prob[i])]}
        t3 = time.perf_counter()
        t["decode"] += t1 - t0
        t["gpu"] += t2 - t1
        t["encode"] += t3 - t2
    with open(os.path.join(output_dir, "top_classes.json"), "w") as f:
        json.dump(top, f, indent=1)
    return written


def build_parser():
    p = argparse.ArgumentParser(description="Render the notebooks' relevance overlays for a folder of images")
    p.add_argument("--images", nargs="+", required=True, help="image files and / or directories of images")
    p.add_argument("--output-dir", required=True)
    p.add_argument("--model", choices=MODELS, default="vit_base_patch16_224")
    p.add_argument("--state-dict", default=None, help="weights with timm key names; pretrained weights are not downloaded")
    p.add_argument("--class-index", type=int, nargs="*", default=[],
                   help="classes explained besides the predicted one (one overlay each)")
    p.add_argument("--use-thresholding", action="store_true", help="Otsu-threshold the relevance first")
    p.add_argument("--transform", choices=("center-crop", "resize"), default=None,
                   help="Resize(256) + CenterCrop(224) (default for the ViT models) or Resize((224, 224)) (default for DeiT)")
    p.add_argument("--batch-size", type=int, default=16)
    p.add_argument("--method", choices=METHODS, default="transformer_attribution",
                   help="the explanation method rendered: transformer_attribution (the notebooks') or the LRP-free "
                        "gradient-weighted attention rollout")
    return p


def parse_args(argv=None):
    p = build_parser()
    args = p.parse_args(argv)
    if args.batch_size < 1:
        p.error("--batch-size must be at least 1")
    if args.transform is None:
        args.transform = "resize" if args.model.startswith("deit") else "center-crop"
    return args


def main(argv=None):
    args = parse_args(argv)
    model = build_model(args.model, args.state_dict)
    if any(not 0 <= c < model.num_classes for c in args.class_index):
        raise SystemExit("--class-index must lie in 0..%d" % (model.num_classes - 1))
    written = run(model, image_paths(args.images), args.output_dir, args.class_index, args.use_thresholding,
                  args.transform, args.batch_size, method=args.method)
    print("%d overlays in %s" % (len(written), args.output_dir))
    return written


if __name__ == "__main__":
    main()
