"""One ViT-B/16 explain step (batch from argv, default 256) at the bench default flags — the target of kernel-filtered ncu captures:
    ncu --set full --clock-control none --import-source on -k regex:wg_kernel -s 8 -c 4 -o prof_attn python tools/profile_step.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformer_explainability_b200 import _lib                                       # noqa: E402
from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224  # noqa: E402

batch = int(sys.argv[1]) if len(sys.argv) > 1 else 256
flags = int(sys.argv[2]) if len(sys.argv) > 2 else _lib.FLAG_BENCH_DEFAULT
torch.manual_seed(0)
m = vit_base_patch16_224().cuda().eval()
x = torch.randn(batch, 3, 224, 224, generator=torch.Generator().manual_seed(1)).cuda()
maps, idx = m.engine().explain(x, flags=flags)
torch.cuda.synchronize()
print(float(maps.abs().max()))
