"""(image, prompt) explanations per second of CLIP image towers on the engine: the gradient-weighted attention rollout of the
image-text similarity (``te_vit_similarity_seed`` + ``TE_FLAG_SIMILARITY_SEED``); prints one JSON line.

    python tools/bench_clip.py [--reps 5] [--warmup 2]

* Towers: ViT-B/32 (N = 50), ViT-B/16 (N = 197) and ViT-L/14 (N = 257) with CLIP's widths (embedding 512 / 512 / 768),
  norm_pre and QuickGELU, random weights (``oracle.clip.init_params(seed=0)``), 224 x 224 inputs resident in HBM, one text
  embedding per image; plus ViT-B/16 with erf GELU at the same shape, so that QuickGELU's cost is visible.
* One step = one engine forward, one seed launch and one ``attribute`` (FLAG_BENCH_DEFAULT | ATTN_GRAD_ROLLOUT |
  SIMILARITY_SEED) at batch 1, 16 and 64: one explanation per image.  Timed with CUDA events, the median of ``--reps``
  rounds after ``--warmup`` warm-up steps.
* ``gpu`` / ``power_limit_w``: the card the numbers were measured on, read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                                             # noqa: E402

from oracle import clip as oclip                                         # noqa: E402
from tools.bench_lrp_rules import _power_limit, _time                    # noqa: E402
from transformer_explainability_b200 import _lib                         # noqa: E402
from transformer_explainability_b200.engine import ViTEngine, vit_config   # noqa: E402

TOWERS = (("clip_vit_b32", dict(patch=32, dim=768, depth=12, heads=12, mlp=3072, embed=512), "quick_gelu"),
          ("clip_vit_b16", dict(patch=16, dim=768, depth=12, heads=12, mlp=3072, embed=512), "quick_gelu"),
          ("clip_vit_l14", dict(patch=14, dim=1024, depth=24, heads=16, mlp=4096, embed=768), "quick_gelu"),
          ("clip_vit_b16_gelu", dict(patch=16, dim=768, depth=12, heads=12, mlp=3072, embed=512), "gelu"))
BATCHES = (1, 16, 64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip.py needs a CUDA device")
    flags = _lib.FLAG_BENCH_DEFAULT
    out = {"gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit(), "flags": flags, "reps": args.reps,
           "cases": {}}
    for name, c, act in TOWERS:
        params, _ = oclip.init_params(seed=0, **c)
        cfg = vit_config(224, c["patch"], 3, c["embed"], c["dim"], c["depth"], c["heads"], c["mlp"] / c["dim"],
                         eps_block=1e-5, eps_final=1e-5, pre_norm=True, act=act)
        eng = ViTEngine(cfg, params, flags=flags)
        rec = {}
        for batch in BATCHES:
            g = torch.Generator().manual_seed(batch)
            x = torch.randn(batch, 3, 224, 224, generator=g).cuda()
            text = torch.randn(batch, c["embed"], generator=g).cuda()

            def step():
                eng.forward(x)
                eng.similarity(text, 100.0)
                eng.attribute(similarity_seeded=True)

            for _ in range(args.warmup):
                step()
            ms = statistics.median(_time(step)[0] for _ in range(args.reps))
            rec["batch_%d" % batch] = {"ms": round(ms, 2), "expl_per_s": round(batch / ms * 1e3, 1)}
        out["cases"][name] = rec
        del eng
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
