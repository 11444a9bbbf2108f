"""Throughput of the perturbation evaluation on one GPU; prints one JSON line.

    python tools/bench_perturbation.py [--batch 64] [--batches 4] [--warmup 1] [--flags BENCH_DEFAULT]

* ``samples_per_s``: samples through ``perturbation.perturbation_eval`` (neg, scale "per": one unperturbed and nine
  perturbed forwards per sample) at ViT-B/16, random-init weights, synthetic inputs resident on the device, after
  ``--warmup`` data batches of the same shape.
* ``perturb_images_ms``: ``te_perturb_images`` alone at the same batch (10 steps), CUDA events over 20 calls, against
  its algorithmic bytes: one read of images and saliency, one write of the 10 x [B,3,224,224] output.
* ``gpu`` / ``power_limit_w``: the card the numbers were measured on, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch                                                             # noqa: E402

HBM_TBPS = 3.35                      # H100 SXM data sheet (700 W)


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                # noqa: BLE001 — reported as unknown, the measurement itself does not depend on it
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--flags", default="BENCH_DEFAULT")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_perturbation needs a CUDA device")
    from transformer_explainability_b200 import _lib, ops, visualization
    from transformer_explainability_b200.baselines.ViT.ViT_new import vit_base_patch16_224
    from transformer_explainability_b200.perturbation import perturbation_eval, perturbation_steps
    torch.manual_seed(0)
    model = vit_base_patch16_224().cuda().eval()
    model.engine_flags = getattr(_lib, "FLAG_" + args.flags) if not args.flags.isdigit() else int(args.flags)
    B = args.batch
    g = torch.Generator(device="cuda").manual_seed(1)

    def batch():
        x = torch.rand(B, 3, 224, 224, device="cuda", generator=g)
        vis = visualization.relevance_to_heatmap(torch.rand(B, 196, device="cuda", generator=g)).reshape(B, 1, 224, 224)
        return x, vis, torch.randint(0, 1000, (B,), device="cuda", generator=g)

    warm = [batch() for _ in range(args.warmup)]
    timed = [batch() for _ in range(args.batches)]
    perturbation_eval(model, warm, neg=True, scale="per")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = perturbation_eval(model, timed, neg=True, scale="per")
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    n = B * args.batches
    assert res["perturbations_hits"].shape == (9, n)

    x, vis, _ = timed[0]
    ks = [0] + perturbation_steps("per")[1]
    s = vis.reshape(B, -1).contiguous()
    for _ in range(3):
        ops.perturb_images(x, s, ks, negate=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps):
        ops.perturb_images(x, s, ks, negate=True)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    P = 224 * 224
    nbytes = (3 + 1) * P * B * 4 + len(ks) * 3 * P * B * 4
    print(json.dumps({
        "metric": "perturbation_eval_samples_per_s", "samples_per_s": round(n / dt, 2), "samples": n, "batch": B,
        "forwards_per_sample": len(ks), "flags": model.engine_flags, "seconds": round(dt, 3),
        "perturb_images_ms": round(ms, 4), "perturb_images_bytes": nbytes,
        "perturb_images_gbps": round(nbytes / ms / 1e6, 1), "perturb_images_frac_of_hbm_datasheet": round(nbytes / ms / 1e9 / HBM_TBPS, 3),
        "gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit()}))


if __name__ == "__main__":
    main()
