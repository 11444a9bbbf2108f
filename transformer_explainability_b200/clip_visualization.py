"""Which patches make each image match each prompt: JET overlays of a CLIP image tower's similarity explanations.

    python -m transformer_explainability_b200.clip_visualization --model-dir DIR --images DIR|FILE... \\
        --text "a dog" "a cat" ... --output-dir OUT [--start-layer N] [--use-thresholding] [--batch-size N]

``--model-dir`` is a local Hugging Face CLIP directory (``clip.CLIPExplainer``).  The prompts are encoded once by the
checkpoint's text tower.  Per batch of images: one resize launch pair per distinct resized size (CLIP's preprocessing:
shorter side to the tower's input size with Pillow's bicubic filter, a center crop, CLIP's mean / std), one engine
forward, and per prompt one seed launch and one ``attribute`` (the gradient-weighted attention rollout of the
similarity), the relevance heatmap at the
model's grid and patch (7 x 32, 14 x 16, 16 x 14) and the notebooks' JET overlay; one device-to-host copy.  Writes
``{stem}_{prompt#}.png`` and ``similarities.json`` ({stem: {"file", "similarities": [one per prompt]}, "prompts": [...]}).
"""
import argparse
import json
import os

import torch

from . import ops
from ._host import to_host
from .visualization import center_crop_geometry, image_paths, relevance_to_heatmap, render_overlays

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def prepare_batch(packed, sizes, offsets, size):
    """CLIP's preprocessing, bit for bit: shorter side to ``size`` (Pillow bicubic), center crop ``size`` x ``size``, CLIP's
    normalisation -> [B, 3, size, size] (device)."""
    geo = [center_crop_geometry(int(h), int(w), size=size, crop=size) for h, w in sizes]
    x = torch.empty(len(sizes), 3, size, size, device=packed.device, dtype=torch.float32)
    groups = {}
    for i, (rs, _) in enumerate(geo):
        groups.setdefault(rs, []).append(i)
    for (rh, rw), idx in groups.items():
        _, y = ops.prepare_images(packed, sizes[idx], offsets[idx], (rh, rw), mean=CLIP_MEAN, std=CLIP_STD, resample="bicubic")
        for j, i in enumerate(idx):
            top, left = geo[i][1]
            x[i] = y[j, :, top:top + size, left:left + size]
    return x


def render_batch(explainer, x, text, start_layer=0, use_thresholding=False):
    """(overlays uint8 [B, P, S, S, 3], similarities [B, P]) on the host for the images x and the P text rows."""
    eng = explainer.engine
    eng.forward(x)
    overlays, sims = [], []
    patch = explainer.kwargs["patch_size"]
    for t in text:
        maps, sim = explainer.explain_forwarded(t, start_layer)
        overlays.append(render_overlays(x, relevance_to_heatmap(maps, grid=explainer.grid, scale=patch), use_thresholding))
        sims.append(sim)
    return to_host(torch.stack(overlays, 1), torch.stack(sims, 1))


def run(explainer, paths, prompts, output_dir, start_layer=0, use_thresholding=False, batch_size=16):
    """The command on parsed arguments; returns the written PNG paths."""
    from PIL import Image
    from . import hdf5_writer
    os.makedirs(output_dir, exist_ok=True)
    dev = explainer.engine.device
    text = explainer.encode_text(prompts).to(dev, torch.float32)
    size = explainer.kwargs["img_size"]
    written, result = [], {"prompts": list(prompts)}
    for s in range(0, len(paths), batch_size):
        chunk = paths[s:s + batch_size]
        packed, sizes, offsets, _ = hdf5_writer.pack_images([(hdf5_writer.read_rgb(p), 0) for p in chunk])
        x = prepare_batch(packed.to(dev), sizes.numpy(), offsets.numpy(), size)
        img, sim = render_batch(explainer, x, text, start_layer, use_thresholding)
        for i, p in enumerate(chunk):
            stem = os.path.splitext(os.path.basename(p))[0]
            for j in range(len(prompts)):
                out = os.path.join(output_dir, "%s_%d.png" % (stem, j))
                Image.fromarray(img[i, j]).save(out)
                written.append(out)
            result[stem] = {"file": os.path.abspath(p), "similarities": [float(v) for v in sim[i]]}
    with open(os.path.join(output_dir, "similarities.json"), "w") as f:
        json.dump(result, f, indent=1)
    return written


def build_parser():
    p = argparse.ArgumentParser(description="Explain a CLIP image tower's image-text similarities as JET overlays")
    p.add_argument("--model-dir", required=True, help="a local Hugging Face CLIP directory (model_type clip)")
    p.add_argument("--images", nargs="+", required=True, help="image files and / or directories of images")
    p.add_argument("--text", nargs="+", required=True, help="the prompts; overlay {stem}_{i}.png explains prompt i")
    p.add_argument("--output-dir", required=True)
    p.add_argument("--start-layer", type=int, default=0)
    p.add_argument("--use-thresholding", action="store_true", help="Otsu-threshold the relevance first")
    p.add_argument("--batch-size", type=int, default=16)
    return p


def parse_args(argv=None):
    p = build_parser()
    args = p.parse_args(argv)
    if args.batch_size < 1:
        p.error("--batch-size must be at least 1")
    if args.start_layer < 0:
        p.error("--start-layer must be at least 0")
    if not os.path.isfile(os.path.join(args.model_dir, "config.json")):
        p.error("--model-dir %s has no config.json" % args.model_dir)
    return args


def main(argv=None):
    from .clip import CLIPExplainer
    args = parse_args(argv)
    explainer = CLIPExplainer(args.model_dir)
    if args.start_layer >= explainer.kwargs["depth"]:
        raise SystemExit("--start-layer must lie in 0..%d" % (explainer.kwargs["depth"] - 1))
    written = run(explainer, image_paths(args.images), args.text, args.output_dir, args.start_layer, args.use_thresholding,
                  args.batch_size)
    print("%d overlays in %s" % (len(written), args.output_dir))
    return written


if __name__ == "__main__":
    main()
