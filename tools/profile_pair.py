"""Launch the persistent pair kernels alone at the four ViT-B shapes (ncu target):
    ncu --set full --clock-control none --import-source on -k regex:wg_kernel -o prof_pair python tools/profile_pair.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformer_explainability_b200 import ops      # noqa: E402

g = torch.Generator(device="cuda").manual_seed(1)
rows = 256 * 197
which = sys.argv[1:] or ["fc2", "fc1"]
for name, inf, outf in [("fc2", 3072, 768), ("fc1", 768, 3072), ("qkv", 768, 2304), ("proj", 768, 768)]:
    if name not in which:
        continue
    x = torch.randn(rows, inf, device="cuda", generator=g)
    w = torch.randn(outf, inf, device="cuda", generator=g) * 0.02
    b = torch.randn(outf, device="cuda", generator=g) * 0.02
    r = torch.rand(rows, outf, device="cuda", generator=g)
    dy = torch.randn(rows, outf, device="cuda", generator=g)
    y = ops.linear_forward(x, w, b, tensor_cores=True)
    ops.linear_relprop(x, w, r, tensor_cores=True, y=y, bias=b)
    ops.linear_backward_tf32(dy, w)
    torch.cuda.synchronize()
    del x, w, b, r, dy, y
