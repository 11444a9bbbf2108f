"""Throughput of the ImageNet-segmentation evaluation on one GPU; prints one JSON line.

    python tools/bench_segmentation.py [--batch 32] [--batches 4] [--warmup 1] [--methods rollout,...]

* ``samples_per_s[method]``: samples through ``segmentation.segmentation_eval`` (explanation + metrics + PR keys; the
  final PR sort and curve included) at ViT-B/16, random-init weights, synthetic images and 0 / 1 masks resident on the
  device, after ``--warmup`` batches of the same shape.
* ``seg_metrics_ms``: ``te_seg_metrics`` alone per batch of 14 x 14 maps (x16 up-sampling, PR keys on), CUDA events.
* ``pr_sort_ms`` / ``pr_curve_ms``: ``te_sort_keys_u32`` and ``te_pr_curve`` over 4276 x 50176 keys (the full data set).
* ``sklearn_host_ms_per_sample``: the reference's host metric calls per sample on the same maps (``average_precision_score``
  over 2 x 50176 scores and ``f1_score`` per image row), when sklearn imports.
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

import numpy as np                                                       # noqa: E402
import torch                                                             # noqa: E402


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                # noqa: BLE001 — reported as unknown, the measurement itself does not depend on it
        return None


def _events(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--methods", type=str, default="rollout,transformer_attribution,full_lrp,lrp_last_layer,"
                                                   "attn_last_layer,attn_gradcam")
    a = ap.parse_args()
    from transformer_explainability_b200 import ops, segmentation as ts
    torch.manual_seed(0)
    B = a.batch
    images = torch.randn(B, 3, 224, 224, device="cuda")
    labels = (torch.rand(B, 224, 224, device="cuda") < 0.4).long()
    out = {"batch": B, "gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit(), "samples_per_s": {}}
    for method in a.methods.split(","):
        lrp, orig_lrp, baselines = ts.build_generators(method)
        run = lambda n: ts.segmentation_eval(method, [(images, labels)] * n, lrp=lrp, orig_lrp=orig_lrp,   # noqa: E731
                                             baselines=baselines)
        run(a.warmup)
        torch.cuda.synchronize()
        t = time.perf_counter()
        run(a.batches)
        torch.cuda.synchronize()
        out["samples_per_s"][method] = round(a.batches * B / (time.perf_counter() - t), 1)
        del lrp, orig_lrp, baselines
        torch.cuda.empty_cache()
    maps = torch.rand(B, 196, device="cuda")
    lab = labels.reshape(B, -1)
    out["seg_metrics_ms"] = round(_events(lambda: ops.seg_metrics(maps, lab, pr_keys=True), 20), 4)
    n = 4276 * 50176
    keys = torch.randint(0, 2 ** 31 - 1, (n,), device="cuda", dtype=torch.int32)
    work = torch.empty_like(keys)
    out["pr_sort_ms"] = round(_events(lambda: ops.sort_keys(keys, out=work), 3), 3)
    out["pr_curve_ms"] = round(_events(lambda: ops.pr_curve(work), 3), 3)
    del keys, work
    try:
        from sklearn.metrics import average_precision_score, f1_score
        m = torch.nn.functional.interpolate(maps[:4].reshape(4, 1, 14, 14).cpu(), scale_factor=16, mode="bilinear")
        t = time.perf_counter()
        for i in range(4):
            r = (m[i, 0] - m[i, 0].min()) / (m[i, 0].max() - m[i, 0].min())
            y = lab[i].cpu().reshape(224, 224)
            onehot = torch.stack([(y == 0), (y == 1)]).reshape(-1).long().numpy()
            average_precision_score(onehot, torch.stack([1 - r, r]).reshape(-1).numpy())
            pred = (r > r.mean()).float().numpy()
            for row in range(224):
                f1_score(y[row].numpy(), pred[row], zero_division=0)
        out["sklearn_host_ms_per_sample"] = round((time.perf_counter() - t) / 4 * 1e3, 1)
    except ImportError:
        out["sklearn_host_ms_per_sample"] = None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
