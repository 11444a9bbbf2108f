"""Time the tensor-core GEMM families alone at the bench shapes (CUDA events, 5 reps after 2 warm-ups):

    python tools/bench_kernels.py            # every family, the default kernel selection

Prints one line per (family, shape): ms, algorithmic TFLOP/s and the fraction of the TF32 roof (measured bf16 / 2).
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformer_explainability_b200 import _lib, ops      # noqa: E402


def timeit(fn, reps=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    rows = int(os.environ.get("ROWS", 256 * 197))
    peak = 850.9
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops"] / 2
    except Exception:
        pass
    g = torch.Generator(device="cuda").manual_seed(1)
    shapes = [("fc2", 3072, 768), ("fc1", 768, 3072), ("qkv", 768, 2304), ("proj", 768, 768)]
    lib = _lib.load()
    for name, inf, outf in shapes:
        x = torch.randn(rows, inf, device="cuda", generator=g)
        w = torch.randn(outf, inf, device="cuda", generator=g) * 0.02
        b = torch.randn(outf, device="cuda", generator=g) * 0.02
        r = torch.rand(rows, outf, device="cuda", generator=g)
        dy = torch.randn(rows, outf, device="cuda", generator=g)
        y = ops.linear_forward(x, w, b, tensor_cores=True)
        ms = timeit(lambda: ops.linear_relprop(x, w, r, tensor_cores=True, y=y, bias=b))
        fl = 8.0 * rows * inf * outf
        print("zplus rule %-5s rows %d in %d out %d: %.3f ms  %.1f TFLOP/s algorithmic = %.3f of TF32 roof (executed 6/8)" % (
            name, rows, inf, outf, ms, fl / ms / 1e9, fl / ms / 1e9 / peak), flush=True)
        ms = timeit(lambda: ops.linear_forward(x, w, b, tensor_cores=True))
        fl = 2.0 * rows * inf * outf
        print("linear fwd 3xTF32 %-5s: %.3f ms  %.1f TFLOP/s algorithmic = %.3f of TF32 roof (x3 issue)" % (
            name, ms, fl / ms / 1e9, fl / ms / 1e9 / peak), flush=True)
        ms = timeit(lambda: ops.linear_forward(x, w, b, tensor_cores=True, f16_split=True))
        print("linear fwd fp16-split %-5s: %.3f ms  %.1f TFLOP/s algorithmic = %.3f of TF32 roof (incl. the row-split pre-pass)" % (
            name, ms, fl / ms / 1e9, fl / ms / 1e9 / peak), flush=True)
        ms = timeit(lambda: ops.linear_backward(dy, w, tensor_cores=True))
        print("linear bwd 3xTF32 %-5s: %.3f ms  %.1f TFLOP/s algorithmic = %.3f of TF32 roof (x3 issue)" % (
            name, ms, fl / ms / 1e9, fl / ms / 1e9 / peak), flush=True)
        if hasattr(ops, "linear_backward_tf32"):
            ms = timeit(lambda: ops.linear_backward_tf32(dy, w))
            print("linear bwd TF32 pair %-5s: %.3f ms  %.1f TFLOP/s = %.3f of TF32 roof" % (
                name, ms, fl / ms / 1e9, fl / ms / 1e9 / peak), flush=True)
        del x, w, b, r, dy, y


if __name__ == "__main__":
    main()
