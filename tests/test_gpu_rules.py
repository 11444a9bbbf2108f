"""GPU: every stand-alone LRP rule through the C ABI vs the oracle and vs the committed reference outputs."""
import os

import numpy as np
import pytest
import torch

from oracle import rules

pytestmark = pytest.mark.gpu


def T(a):
    return torch.from_numpy(np.asarray(a))


def dev(t):
    return t.to("cuda", torch.float32).contiguous()


def rel_err(a, b):
    b = b.double()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


@pytest.fixture(scope="module")
def ops():
    from transformer_explainability_b200 import ops as o
    return o


def test_golden_rules_on_gpu(ops, golden_dir):
    g = np.load(os.path.join(golden_dir, "rules.npz"))
    out = ops.linear_relprop(dev(T(g["lin_x"])), dev(T(g["lin_w"])), dev(T(g["lin_r"])))
    assert rel_err(out, T(g["lin_out"])) < 2e-5
    oa, ob = ops.add_relprop(dev(T(g["add_a"])), dev(T(g["add_b"])), dev(T(g["add_r"])))
    assert rel_err(oa, T(g["add_oa"])) < 1e-4 and rel_err(ob, T(g["add_ob"])) < 1e-4
    out = ops.clone_relprop(dev(T(g["clone_x"])), [dev(T(g["clone_r1"])), dev(T(g["clone_r2"]))])
    assert rel_err(out, T(g["clone_out"])) < 1e-6
    op, ov = ops.matmul_av_relprop(dev(T(g["av_p"])), dev(T(g["av_v"])), dev(T(g["av_r"])))
    assert rel_err(op, T(g["av_op"])) < 1e-3 and rel_err(ov, T(g["av_ov"])) < 1e-3
    oq, ok = ops.matmul_qk_relprop(dev(T(g["qk_q"])), dev(T(g["qk_k"])), dev(T(g["qk_r"])))
    assert rel_err(oq, T(g["qk_oq"])) < 1e-3 and rel_err(ok, T(g["qk_ok"])) < 1e-3
    out = ops.index_select_relprop(dev(T(g["isel_x"])), dev(T(g["isel_r"])))
    assert rel_err(out, T(g["isel_out"])) < 1e-6


@pytest.mark.parametrize("rows,inf,outf", [(197, 768, 768), (130, 64, 256), (64, 3072, 768), (5, 768, 1000),
                                           (333, 192, 64), (2955, 768, 3072), (3001, 3072, 768), (2048, 768, 2304)])
def test_linear_forward_and_relprop(ops, rows, inf, outf):
    g = torch.Generator().manual_seed(rows + inf)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    b = torch.randn(outf, generator=g)
    r = torch.rand(rows, outf, generator=g)
    y = ops.linear_forward(dev(x), dev(w), dev(b))
    assert rel_err(y, torch.nn.functional.linear(x.double(), w.double(), b.double())) < 5e-6
    out = ops.linear_relprop(dev(x), dev(w), dev(r))
    ref = rules.linear_relprop(x.double(), w.double(), r.double())
    assert rel_err(out, ref) < 2e-5          # Z is a sum of non-negative products: well conditioned
    # conservation: sum of relevance is preserved by the z+ rule (ViT_LRP.py:326,334 comments)
    assert abs(out.double().sum().item() - r.double().sum().item()) < 1e-4 * r.sum().item()


@pytest.mark.parametrize("b,n,d", [(1, 197, 768), (3, 17, 64), (2, 512, 768)])
def test_add_and_clone(ops, b, n, d):
    g = torch.Generator().manual_seed(b * n)
    x1 = torch.randn(b, n, d, generator=g)
    x2 = torch.randn(b, n, d, generator=g) + 0.5
    r = torch.randn(b, n, d, generator=g)
    r1, r2 = ops.add_relprop(dev(x1), dev(x2), dev(r))
    # fp32 oracle with fp64 sums is what the kernel computes; signed Z ~ 0 makes this rule ill-conditioned,
    # so compare against the fp32 formula evaluated on the SAME fp32 inputs, elementwise part in fp32
    s = rules.safe_divide(r, x1 + x2)
    a, bb = x1 * s, x2 * s
    A, B_, rho = [t.double().reshape(b, -1).sum(1).reshape(b, 1, 1) for t in (a, bb, r)]
    den = A.abs() + B_.abs()
    fa = rules.safe_divide(rules.safe_divide(A.abs(), den) * rho, A).float()
    fb = rules.safe_divide(rules.safe_divide(B_.abs(), den) * rho, B_).float()
    assert rel_err(r1, a * fa) < 1e-5 and rel_err(r2, bb * fb) < 1e-5
    # conservation per sample: sum(r1)+sum(r2) == sum(r)
    tot = (r1.double().reshape(b, -1).sum(1) + r2.double().reshape(b, -1).sum(1)).cpu()
    assert torch.allclose(tot, r.double().reshape(b, -1).sum(1), rtol=1e-4, atol=1e-4)
    out = ops.clone_relprop(dev(x1), [dev(r), dev(x2)])
    assert rel_err(out, rules.clone_relprop(x1, (r, x2))) < 1e-6
    out3 = ops.clone_relprop(dev(x1), [dev(r), dev(x2), dev(x1 * 0.3)])
    assert rel_err(out3, rules.clone_relprop(x1, (r, x2, x1 * 0.3))) < 1e-6


@pytest.mark.parametrize("b,h,n,d", [(2, 12, 197, 64), (1, 4, 17, 16), (1, 2, 512, 64), (2, 3, 198, 64)])
def test_attention_matmul_rules(ops, b, h, n, d):
    g = torch.Generator().manual_seed(n)
    p = torch.randn(b, h, n, n, generator=g).softmax(-1)
    v = torch.randn(b, h, n, d, generator=g)
    q = torch.randn(b, h, n, d, generator=g)
    k = torch.randn(b, h, n, d, generator=g)
    # relevance proportional to Z^2 makes S = R/Z = Z*u continuous through Z = 0, so that fp32-vs-fp64 sign flips
    # of a near-zero Z do not dominate the comparison (the rule itself is ill-conditioned for signed Z)
    r_av = (p @ v) ** 2 * torch.rand(b, h, n, d, generator=g)
    r_qk = (q @ k.transpose(-1, -2)) ** 2 * torch.rand(b, h, n, n, generator=g)
    rp, rv = ops.matmul_av_relprop(dev(p), dev(v), dev(r_av))
    op, ov = rules.matmul_av_relprop(p.double(), v.double(), r_av.double())
    assert rel_err(rp, op) < 1e-4 and rel_err(rv, ov) < 1e-4
    rq, rk = ops.matmul_qk_relprop(dev(q), dev(k), dev(r_qk))
    oq, ok = rules.matmul_qk_relprop(q.double(), k.double(), r_qk.double())
    assert rel_err(rq, oq) < 1e-4 and rel_err(rk, ok) < 1e-4


@pytest.mark.parametrize("B,C,S,P,D", [(2, 3, 32, 8, 64), (3, 3, 224, 16, 768), (1, 3, 48, 16, 40)])
def test_patch_embed_zb_rule(ops, B, C, S, P, D):
    """Conv2d.relprop z^B branch behind PatchEmbed.relprop (layers_ours.py:242-259) vs the fp64 restatement."""
    g = torch.Generator().manual_seed(S + D)
    img = torch.randn(B, C, S, S, generator=g)
    w = torch.randn(D, C, P, P, generator=g) * 0.05
    r = torch.randn(B, (S // P) ** 2, D, generator=g)
    ref = rules.conv_zb_relprop(img.double(), w.double(), r.transpose(1, 2).reshape(B, D, S // P, S // P).double(), P)
    out = ops.patch_embed_relprop(dev(img), dev(w), dev(r))
    assert out.shape == ref.shape
    assert rel_err(out, ref) < 2e-5
    out_sum = ops.patch_embed_relprop(dev(img), dev(w), dev(r), per_channel=False)
    assert rel_err(out_sum, ref.sum(dim=1)) < 2e-5
    # the reference-shaped layer class (modules.layers_ours.Conv2d: forward hook stashes X, relprop(R, alpha))
    from transformer_explainability_b200.modules import layers_ours as L
    conv = L.Conv2d(C, D, kernel_size=P, stride=P).cuda()
    with torch.no_grad():
        conv.weight.copy_(w)
    conv(dev(img))
    r_conv = dev(r).transpose(1, 2).reshape(B, D, S // P, S // P).contiguous()
    assert rel_err(conv.relprop(r_conv, alpha=1), ref) < 2e-5
    # conservation: sum of the pixel relevance == sum of R * (Za - 1e-9) / Za ~= sum R
    assert abs(out.double().sum().item() - r.double().sum().item()) < 1e-3 * r.abs().double().sum().item()


@pytest.mark.parametrize("L,B,H,N,normalize", [(12, 2, 12, 197, False), (3, 3, 4, 17, False), (4, 1, 12, 512, True),
                                               (12, 2, 12, 198, False), (2, 40, 16, 197, True), (12, 300, 2, 30, False),
                                               (3, 3, 2, 301, True)])
def test_aggregation_rollout(ops, L, B, H, N, normalize):
    g = torch.Generator().manual_seed(N + L)
    grad = torch.randn(L, B, H, N, N, generator=g) * 0.05
    cam = torch.randn(L, B, H, N, N, generator=g) * 0.05
    for start in (0, 1, L - 1):
        mats = [rules.aggregate(grad[l].double(), cam[l].double()) for l in range(L)]
        ref = rules.rollout(mats, start_layer=start, normalize=normalize)
        joint, row0 = ops.attribution_rollout(dev(grad), dev(cam), start_layer=start, normalize=normalize)
        assert rel_err(joint, ref) < 1e-5
        assert rel_err(row0, ref[:, 0]) < 1e-5
        # fused single-kernel row-only path (what generate_LRP consumes)
        _, row_f = ops.attribution_rollout(dev(grad), dev(cam), start_layer=start, normalize=normalize, fused=True,
                                           want_joint=False)
        assert rel_err(row_f, ref[:, 0]) < 1e-5
        # dense joint with the fast flag: N x N x N chain on the tensor cores (3xTF32)
        joint_tc, row_tc = ops.attribution_rollout(dev(grad), dev(cam), start_layer=start, normalize=normalize,
                                                   fused=True, want_joint=True)
        assert rel_err(joint_tc, ref) < 1e-5 and rel_err(row_tc, ref[:, 0]) < 1e-5
        assert (joint_tc.cpu().double() - ref).abs().max() < 2e-6 * max(1.0, ref.abs().max().item())
        off = ~torch.eye(N, dtype=torch.bool)                    # the small off-diagonal entries, relative to themselves
        assert ((joint_tc.cpu().double() - ref).abs()[:, off].max() / ref[:, off].abs().max()).item() < 2e-5
        # public compute_rollout_attention on pre-aggregated matrices
        j2 = ops.compute_rollout_attention([dev(m.float()) for m in mats], start_layer=start, normalize=normalize)
        assert rel_err(j2, ref) < 1e-5
