"""Launch the kernels the roofline is quoted on, alone, at the bench shapes — the target of the ncu captures:

    ncu --set full --clock-control none --import-source on -k regex:wg_kernel -c 2 -o prof_tc \
        python tools/profile_kernels.py zplus_tc
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformer_explainability_b200 import ops      # noqa: E402


def main():
    what = sys.argv[1]
    g = torch.Generator(device="cuda").manual_seed(1)
    if what == "zplus_tc_s1":                     # what the engines run: single-pass S kernel (saved forward output) + R kernel
        rows, inf, outf = 256 * 197, 3072, 768
        x = torch.randn(rows, inf, device="cuda", generator=g)
        w = torch.randn(outf, inf, device="cuda", generator=g) * 0.02
        b = torch.randn(outf, device="cuda", generator=g) * 0.1
        r = torch.rand(rows, outf, device="cuda", generator=g)
        y = ops.linear_forward(x, w, b, tensor_cores=True)
        for _ in range(2):
            ops.linear_relprop(x, w, r, tensor_cores=True, y=y, bias=b)
    elif what in ("zplus_tc", "zplus_simt"):
        rows, inf, outf = 256 * 197, 3072, 768
        x = torch.randn(rows, inf, device="cuda", generator=g)
        w = torch.randn(outf, inf, device="cuda", generator=g) * 0.02
        r = torch.rand(rows, outf, device="cuda", generator=g)
        for _ in range(2):
            ops.linear_relprop(x, w, r, tensor_cores=(what == "zplus_tc"))
    elif what in ("rollout", "rollout_fused"):
        L, B, H, N = 12, 32, 12, 197
        grad = torch.randn(L, B, H, N, 200, device="cuda", generator=g) * 0.05
        cam = torch.randn(L, B, H, N, 200, device="cuda", generator=g) * 0.05
        for _ in range(2):
            ops.attribution_rollout(grad, cam, fused=(what == "rollout_fused"), want_joint=False)
    elif what == "linear_fwd":
        rows, inf, outf = 256 * 197, 768, 3072
        x = torch.randn(rows, inf, device="cuda", generator=g)
        w = torch.randn(outf, inf, device="cuda", generator=g) * 0.02
        b = torch.randn(outf, device="cuda", generator=g)
        for _ in range(2):
            ops.linear_forward(x, w, b)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
