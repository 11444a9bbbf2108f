"""Where one bench step's GPU time goes: one warmed ViT-B/16 explain step (bench.py's workload: batch 256, flags 7475,
resident inputs) under torch.profiler, kernel time summed per kernel name and per tensor-core problem family.

    python tools/profile_step_kernels.py [--batch 256] [--flags 7475] [--top 25]

The profiler slows the host, so the printed step time is not a throughput figure (bench.py is).
"""
import argparse
import collections
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformer_explainability_b200 import _lib                                       # noqa: E402
from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224  # noqa: E402


def family(name):
    """'wg_kernel<LinProb<2, 2> >' -> 'LinProb<2, 2>' ; other kernels keep their base name."""
    n = name.replace("(anonymous namespace)::", "")
    m = re.search(r"wg_kernel<(\w+<[^>]*>)", n)
    if m:
        return m.group(1)
    return re.sub(r"\(.*$", "", n).replace("void ", "").strip()


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the card name still comes from torch
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--flags", type=int, default=_lib.FLAG_BENCH_DEFAULT)
    ap.add_argument("--top", type=int, default=25)
    args = ap.parse_args()
    _lib.load()
    print("card:", card(), flush=True)
    torch.manual_seed(0)
    eng = vit_base_patch16_224(pretrained=False).cuda().eval().engine()
    x = torch.randn(args.batch, 3, 224, 224, generator=torch.Generator().manual_seed(1)).cuda()
    for _ in range(2):
        eng.explain(x, flags=args.flags, chunk=args.batch)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.profiler.profile(activities=acts) as prof:
        e0.record()
        eng.explain(x, flags=args.flags, chunk=args.batch)
        e1.record()
        torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1)
    per_name, per_family = collections.Counter(), collections.Counter()
    calls = collections.Counter()
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        per_name[ev.name] += us
        per_family[family(ev.name)] += us
        calls[ev.name] += 1
    kern_ms = sum(per_name.values()) / 1e3
    print("flags=%d batch=%d: step %.1f ms (under the profiler), kernel time %.1f ms" % (args.flags, args.batch, step_ms, kern_ms))
    print("\nper family (kernel ms, share of the step):")
    for name, us in per_family.most_common(args.top):
        print("  %9.2f ms  %5.1f %%  %s" % (us / 1e3, 100.0 * us / 1e3 / step_ms, name))
    print("\nper kernel name (kernel ms, share of the step, launches):")
    for name, us in per_name.most_common(args.top):
        print("  %9.2f ms  %5.1f %%  %4d  %s" % (us / 1e3, 100.0 * us / 1e3 / step_ms, calls[name], name[:160]))
    linear = ("LinProb", "ZsProb", "ZrProb")
    share = sum(us for n, us in per_family.items() if n.startswith(linear)) / 1e3
    print("\nLinear-rule GEMMs (%s): %.1f ms = %.1f %% of the step" % (" + ".join(linear), share, 100.0 * share / step_ms))


if __name__ == "__main__":
    main()
