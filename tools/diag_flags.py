"""GPU diagnostic (VERDICT r01 task 1d): which kernel selection costs map accuracy on the ill-conditioned random-init
ViT-B?  For samples 0..3, 32 copies of the input perturbed by 1e-7 relative noise; per flag set the quartiles of the map
error vs the fp64 oracle, beside the fp32 CPU oracle (== the reference, bit-equal) evaluated on the SAME perturbed
inputs.  A selection is "in the reference's noise class" when its quartiles match the CPU fp32 column.

    python tools/diag_flags.py [trials] > flag_bisect.log
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import vit as ovit, cpu as ocpu          # noqa: E402
from transformer_explainability_b200 import _lib    # noqa: E402
from transformer_explainability_b200.baselines.ViT.ViT_LRP import vit_base_patch16_224  # noqa: E402


def quart(errs):
    e = sorted(errs)
    n = len(e)
    return e[n // 4], 0.5 * (e[n // 2 - 1] + e[n // 2]), e[(3 * n) // 4]


def main():
    trials = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    ocpu.set_torch_threads()
    params, heads = ovit.init_params("vit_base_patch16_224", seed=0)
    xs0 = torch.randn(8, 3, 224, 224, generator=torch.Generator().manual_seed(100))
    m = vit_base_patch16_224()
    m.load_state_dict(params)
    m = m.cuda().eval()
    eng = m.engine()
    p64 = {k: v.double() for k, v in params.items()}
    F = _lib
    sets = [("fp32 SIMT (0)", 0), ("+z+ TF32 (1)", 1), ("+3xTF32 linears (17)", 17), ("+3xTF32 attention (33)", 33),
            ("all r01 (51)", 51), ("linears + TF32 backward (273)", 273), ("bench default (%d)" % F.FLAG_BENCH_DEFAULT, F.FLAG_BENCH_DEFAULT)]
    print("ViT-B/16 random init, %d copies of each input with 1e-7 relative noise; map L_inf error / map max vs the fp64 oracle of "
          "the unperturbed input: lower quartile / median / upper quartile" % trials)
    for sample in range(4):
        x0 = xs0[sample:sample + 1]
        xb = torch.cat([x0] + [x0 * (1 + 1e-7 * torch.randn(x0.shape, generator=torch.Generator().manual_seed(100 + k)))
                               for k in range(1, trials)])
        ref0, _ = ovit.explain(p64, x0.double(), heads)
        sc = ref0.abs().max().item()
        cpu32 = [(ovit.explain(params, xb[k:k + 1], heads)[0].double() - ref0).abs().max().item() / sc for k in range(trials)]
        print("sample %d  %-34s q1 %.1e  med %.1e  q3 %.1e" % ((sample, "CPU fp32 oracle (= reference)") + quart(cpu32)), flush=True)
        for name, fl in sets:
            maps, _ = eng.explain(xb.cuda(), flags=fl)
            errs = [(maps[k].cpu().double() - ref0[0]).abs().max().item() / sc for k in range(trials)]
            print("sample %d  %-34s q1 %.1e  med %.1e  q3 %.1e" % ((sample, name) + quart(errs)), flush=True)


if __name__ == "__main__":
    main()
