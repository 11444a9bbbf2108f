"""Write the output of every Linear-rule tensor-core op at the ViT-B/16 bench shapes (batch 256: 50432 token rows) from
seeded inputs, one .npy per op, so that two builds can be compared byte for byte (e.g. with ``cmp``):

    python tools/dump_linear_ops.py OUT_DIR

Ops: the fp16-split forward (fc1), the single-pass TF32 and fp16 backward (fc2), and Linear.relprop at the fc2 shape in
every tensor-core form (bf16 / TF32 single-pass denominator, fp32 / bf16 / fp16 second contraction, alpha-beta, the
layers_lrp rule).  Then the attention-shaped contractions of one attention block with the operand forms of the bench flags
(``ops.tc_attention_nn`` / ``ops.tc_attention_nk``: softmax, P V, dctx V^T, P^T dctx, dS K, dS^T Q, the MUL and SD
epilogues of the relevance side) at batch 32 x 12 heads, N = 197, maps padded to 200 columns, and the dense rollout joint
(``ops.attribution_rollout(..., fused=True, want_joint=True)``).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from transformer_explainability_b200 import ops  # noqa: E402

ROWS, D, MLP = 256 * 197, 768, 3072


def rand(seed, *shape, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g) * scale


def main():
    out_dir = sys.argv[1]
    os.makedirs(out_dir, exist_ok=True)

    def save(name, t):
        torch.cuda.synchronize()
        np.save(os.path.join(out_dir, name + ".npy"), t.cpu().numpy())
        print(name, tuple(t.shape), flush=True)

    x, w1, b1 = rand(1, ROWS, D), rand(2, MLP, D, scale=D ** -0.5), rand(3, MLP, scale=0.1)
    save("fwd_f16_split", ops.linear_forward_epi(x, w1, b1, epi="bias", family="f16_split")[0])
    w2 = rand(4, D, MLP, scale=MLP ** -0.5)
    dy = rand(5, ROWS, D)
    save("bwd_tf32", ops.linear_backward_tf32(dy, w2))
    save("bwd_f16", ops.linear_backward_epi(dy, w2, epi="store", family="f16"))
    del x, dy

    h, b2 = rand(6, ROWS, MLP), rand(7, D, scale=0.1)
    r = rand(8, ROWS, D).abs_()
    y = ops.linear_forward(h, w2, b2)
    forms = {"bf16_s1": dict(bf16="s1"), "tf32": {}, "f16_r": dict(bf16="s1", r_f16=True), "f16_r_tf32": dict(r_f16=True),
             "bf16_r": dict(bf16=True)}
    for name, kw in forms.items():
        save("relprop_" + name, ops.linear_relprop(h, w2, r, tensor_cores=True, y=y, bias=b2, **kw))
    save("relprop_bf16_s1_alpha2", ops.linear_relprop(h, w2, r, tensor_cores=True, y=y, bias=b2, bf16="s1", alpha=2.0))
    save("relprop_lrp_tc", ops.linear_relprop(h, w2, r, variant="lrp_tc"))
    save("relprop_lrp_tc_alpha2", ops.linear_relprop(h, w2, r, variant="lrp_tc", alpha=2.0))
    del h, r, y

    B, H, N, NP = 32, 12, 197, 200
    qkv, act = rand(9, B * N, 3 * D), rand(10, B * N, D)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    emap = torch.nn.functional.pad(rand(11, B, H, N, N).abs_() + 0.5, (0, NP - N)).contiguous()

    def nn(a, b, epi, sp, e=None):
        out = torch.empty(B, H, N, NP, device="cuda")
        return ops.tc_attention_nn(a, a.stride(0), b, b.stride(0), B, H, N, 64, out, NP, e=e, alpha=0.125, epi=epi, single_pass=sp)

    def nk(amap, amn, x, epi, sp, e=None):
        out = torch.empty(B * N, D, device="cuda")
        return ops.tc_attention_nk(amap, NP, amn, x, x.stride(0), B, H, N, out, D, e=e, alpha=0.5, epi=epi, single_pass=sp)

    p = nn(q, k, "softmax", False)
    save("attn_softmax", p)
    save("attn_pv", nk(p, 0, v, "store", False))
    save("attn_g", nn(act, v, "store", True))
    save("attn_dv", nk(p, 1, act, "store", True))
    save("attn_dq", nk(emap, 0, k, "store", True))
    save("attn_dk", nk(emap, 1, q, "store", True))
    save("attn_cam", nn(act, v, "mul", True, e=p))
    save("attn_rv", nk(p, 1, act, "mul", True, e=act))
    save("attn_s1", nn(q, k, "sd", False, e=emap))
    save("attn_rq", nk(emap, 0, k, "mul", True, e=act))
    save("attn_nn_store_3x", nn(q, k, "store", False))
    save("attn_nn_mul_3x", nn(act, v, "mul", False, e=emap))
    save("attn_nk_mul_3x", nk(emap, 1, v, "mul", False, e=act))
    grad, cam = rand(12, 12, 8, H, N, NP, scale=0.05), rand(13, 12, 8, H, N, NP, scale=0.05)
    save("rollout_dense_joint", ops.attribution_rollout(grad, cam, fused=True, want_joint=True)[0])


if __name__ == "__main__":
    main()
