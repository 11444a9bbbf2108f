"""The attention-shaped contractions on the TMA mainloop (``NnProb`` / ``NkProb`` in te_tc_wgmma.cu, persistent CTAs walking
sample x head x tile, operands TF32-rounded, split into hi / lo and transposed in shared memory): every instantiation the ops
API reaches, and the dense rollout chain (``NkProb<0, AT_RESID>``), at token counts around the tile edges and at
(batch, heads) giving fewer tiles than SMs and tile counts that are not a multiple of the grid.

Each case must be deterministic (two runs bit-equal), position-independent (sample 0 run alone in a batch-1 launch, where
it falls on another CTA and at another phase of the stage ring, and its ragged tile reads zeros instead of sample 1's rows,
equals its slice of the full launch bit for bit) and within the fp64 bounds of tests/test_gpu_attention_tc.py."""
import math

import pytest
import torch

from oracle import rules
from transformer_explainability_b200 import ops

pytestmark = pytest.mark.gpu

NS = [1, 17, 128, 129, 197, 256, 300, 512]
BH = [(1, 1), (3, 12), (37, 12)]
BOUND_SP = 2e-3


def bound_3x(K):
    return 1.5e-8 * K + 2e-6


def npad(n):
    return (n + 3) & ~3


def bits(t):
    return t.contiguous().view(torch.int32)


def per_element(out, ref, scale):
    out = out.double()
    live = scale > 0
    assert (out[~live] == ref[~live]).all()
    return ((out - ref).abs()[live] / scale[live]).max().item() if live.any() else 0.0


def heads_of(rows, batch, heads, n, dh):
    return rows.double().reshape(batch, n, heads, dh).permute(0, 2, 1, 3)


def check(run, batch, part):
    """run(b0, nb) -> output of samples b0 .. b0 + nb - 1; two full runs bit-equal, sample 0 alone bit-equal to its slice"""
    a, b = run(0, batch), run(0, batch)
    torch.cuda.synchronize()
    assert torch.equal(bits(a), bits(b)), "two runs differ"
    one = run(0, 1)
    torch.cuda.synchronize()
    assert torch.equal(bits(one), bits(part(a))), "sample 0 differs when run alone"
    return a


@pytest.mark.parametrize("batch,heads", BH)
@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("n", NS)
def test_nn(n, dh, batch, heads):
    """out = epi(alpha q k^T): STORE / MUL in single-pass and 3xTF32 form, SD, and the fused SOFTMAX (N <= 256)"""
    D = heads * dh
    g = torch.Generator(device="cuda").manual_seed(n * 31 + dh + batch)
    qkv = torch.randn(batch * n, 3 * D, generator=g, device="cuda")
    ld = npad(n)
    E = torch.rand(batch, heads, n, ld, generator=g, device="cuda") + 0.5
    q, k = heads_of(qkv[:, :D], batch, heads, n, dh), heads_of(qkv[:, D:2 * D], batch, heads, n, dh)
    s64, a64 = torch.einsum("bhid,bhjd->bhij", q, k), torch.einsum("bhid,bhjd->bhij", q.abs(), k.abs())
    alpha = float(torch.tensor(1.0 / math.sqrt(dh)))

    def run(epi, sp, e=None):
        def f(b0, nb):
            out = torch.empty(nb, heads, n, ld, device="cuda")
            rows = qkv[b0 * n:(b0 + nb) * n]
            ops.tc_attention_nn(rows, 3 * D, rows[:, D:], 3 * D, nb, heads, n, dh, out, ld,
                                None if e is None else e[b0:b0 + nb].contiguous(), alpha, epi, sp)
            return out
        return check(f, batch, lambda t: t[:1])

    e64 = E[..., :n].double()
    for sp in (False, True):
        out = run("store", sp)
        assert (out[..., n:] == 0).all()
        err = per_element(out[..., :n], alpha * s64, alpha * a64)
        assert err < (BOUND_SP if sp else bound_3x(dh)), "store sp=%s: %g" % (sp, err)
        out = run("mul", sp, E)
        err = per_element(out[..., :n], alpha * s64 * e64, alpha * a64 * e64)
        assert err < (BOUND_SP if sp else bound_3x(dh)), "mul sp=%s: %g" % (sp, err)
    z = run("store", False)
    sd = run("sd", False, E)
    ref = rules.safe_divide(e64, z[..., :n].double())
    assert ((sd[..., :n].double() - ref).abs() / ref.abs().clamp_min(1e-300)).max().item() < 4e-7
    if n <= 256:
        p = run("softmax", False)[..., :n].double()
        ref = torch.softmax(alpha * s64, dim=-1)
        live = ref > 1e-30
        bound = (2 * alpha * a64.amax(dim=-1, keepdim=True) * bound_3x(dh) + 1e-5).expand_as(ref)
        assert (((p - ref).abs() / ref.clamp_min(1e-300))[live] < bound[live]).all()


@pytest.mark.parametrize("batch,heads", BH)
@pytest.mark.parametrize("amn", [0, 1])
@pytest.mark.parametrize("n", NS)
def test_nk(n, amn, batch, heads):
    """out = epi(alpha M_h x_h) with M_h the map (amn 0) or its transpose (amn 1): STORE / MUL, single pass and 3xTF32;
    NaN in the map's padding columns is never read"""
    D, np_ = heads * 64, npad(n)
    g = torch.Generator(device="cuda").manual_seed(n * 37 + amn + batch)
    qkv = torch.randn(batch * n, 3 * D, generator=g, device="cuda")
    amap = torch.full((batch, heads, n, np_), float("nan"), device="cuda")
    amap[..., :n] = torch.randn(batch, heads, n, n, generator=g, device="cuda")
    E = torch.rand(batch * n, D, generator=g, device="cuda") + 0.5
    m = amap[..., :n].double()
    if amn:
        m = m.transpose(-1, -2)
    v = heads_of(qkv[:, 2 * D:], batch, heads, n, 64)
    ref = (0.5 * m @ v).permute(0, 2, 1, 3).reshape(batch * n, D)
    scale = (0.5 * m.abs() @ v.abs()).permute(0, 2, 1, 3).reshape(batch * n, D)

    for epi in ("store", "mul"):
        for sp in (False, True):
            def f(b0, nb, epi=epi, sp=sp):
                out = torch.empty(nb * n, D, device="cuda")
                rows = qkv[b0 * n:(b0 + nb) * n]
                ops.tc_attention_nk(amap[b0:b0 + nb], np_, amn, rows[:, 2 * D:], 3 * D, nb, heads, n, out, D,
                                    E[b0 * n:(b0 + nb) * n] if epi == "mul" else None, 0.5, epi, sp)
                return out
            out = check(f, batch, lambda t: t[:n])
            e = E.double() if epi == "mul" else 1.0
            err = per_element(out, ref * e, scale * e)
            assert err < (BOUND_SP if sp else bound_3x(n)), "%s sp=%s: %g" % (epi, sp, err)


@pytest.mark.parametrize("L,B,H,N,normalize", [(3, 1, 12, 17, False), (3, 3, 12, 197, False), (2, 37, 4, 129, True),
                                               (3, 2, 12, 300, False)])
def test_dense_rollout(L, B, H, N, normalize):
    """the dense joint of attribution_rollout(fused=True, want_joint=True): the chain J <- A_l J + d_l * J on NkProb<0, RESID>"""
    g = torch.Generator(device="cuda").manual_seed(N + L + B)
    np_ = npad(N)
    grad = torch.zeros(L, B, H, N, np_, device="cuda")
    cam = torch.zeros(L, B, H, N, np_, device="cuda")
    grad[..., :N] = torch.randn(L, B, H, N, N, generator=g, device="cuda") * 0.05
    cam[..., :N] = torch.randn(L, B, H, N, N, generator=g, device="cuda") * 0.05

    def f(b0, nb):
        return ops.attribution_rollout(grad[:, b0:b0 + nb].contiguous(), cam[:, b0:b0 + nb].contiguous(), normalize=normalize,
                                       fused=True, want_joint=True)[0]
    joint = check(f, B, lambda t: t[:1])
    mats = [rules.aggregate(grad[l, ..., :N].double().cpu(), cam[l, ..., :N].double().cpu()) for l in range(L)]
    ref = rules.rollout(mats, start_layer=0, normalize=normalize)
    assert (joint.cpu().double() - ref).abs().max() < 2e-6 * max(1.0, ref.abs().max().item())
