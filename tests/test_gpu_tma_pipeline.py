"""The Linear-rule GEMMs fed by TMA on persistent CTAs (``wg_kernel`` problems with ``P::TMA`` in te_tc_wgmma.cu): every
family through the ops API at shapes that stress the stage ring and the tile walk — fewer k-blocks than stages, k-block
counts that are not a multiple of the stage count, single and partial row tiles, fewer tiles than SMs and tile counts that
are not a multiple of the grid, and the accumulating inhibitor half of the alpha-beta rule.

Each case must be deterministic (two runs bit-equal), position-independent (rows recomputed in a launch of just their
neighbourhood, where they sit in another tile, on another CTA and at another phase of the ring, are bit-equal) and within
the family's fp64 bound."""
import pytest
import torch

from oracle import alphabeta
from transformer_explainability_b200 import ops

pytestmark = pytest.mark.gpu

TF32, BF16_R = 3e-3, 1.5e-2


def rel(a, b):
    b = b.double().cpu()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def inputs(seed, *shapes):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(*s, generator=g) for s in shapes]


def check_rows(fn, row_inputs, ref, bound):
    """fn(*row_inputs) twice (bit-equal), around its first / middle / last row (bit-equal), and against ref"""
    rows = row_inputs[0].shape[0]
    a, b = fn(*row_inputs), fn(*row_inputs)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two runs differ"
    for r in sorted({0, rows // 2, rows - 1}):
        sl = slice(max(0, r - 3), min(rows, r + 4))
        part = fn(*(t[sl].contiguous() for t in row_inputs))
        assert torch.equal(part.view(torch.int32), a[sl].contiguous().view(torch.int32)), "rows %s differ in a short launch" % sl
    e = rel(a, ref)
    assert e < bound, "rel err %g" % e


# (rows, K, N): K = 64 / 32 (fewer k-blocks than stages), 384 and 3072 (not a multiple of the stage count); rows 1, 127,
# 129 (one and two row tiles, few CTAs) and 20000 (157 row tiles: more tiles than SMs, not a multiple of the grid)
LIN_SHAPES = [(1, 64, 128), (127, 384, 256), (129, 3072, 128), (20000, 384, 768)]


@pytest.mark.parametrize("rows,K,N", LIN_SHAPES)
def test_f16_split_forward(rows, K, N):                             # LinProb<BIAS, LIN_F16X3>
    x, w, b = inputs(rows + K, (rows, K), (N, K), (N,))
    w *= K ** -0.5
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    ref = x.double() @ w.double().t() + b.double()
    check_rows(lambda xx: ops.linear_forward_epi(xx, wd, bd, epi="bias", family="f16_split")[0], [xd], ref, TF32)


@pytest.mark.parametrize("rows,K,N", [(1, 32, 128)] + LIN_SHAPES)
def test_tf32_backward(rows, K, N):                                 # LinProb<STORE, LIN_TF32>: A rounded in shared memory
    dy, w = inputs(rows + K + 1, (rows, K), (K, N))
    w *= K ** -0.5
    wd = w.cuda()
    check_rows(lambda d: ops.linear_backward_tf32(d, wd), [dy.cuda()], dy.double() @ w.double(), TF32)


@pytest.mark.parametrize("rows,K,N", LIN_SHAPES)
def test_f16_backward(rows, K, N):                                  # LinProb<STORE, LIN_F16>
    dy, w = inputs(rows + K + 2, (rows, K), (K, N))
    w *= K ** -0.5
    wd = w.cuda()
    check_rows(lambda d: ops.linear_backward_epi(d, wd, epi="store", family="f16"), [dy.cuda()], dy.double() @ w.double(), TF32)


# (name, ops.linear_relprop kwargs, bound): the S kernel and the R kernel each family runs
RULES = [("bf16_s1", dict(tensor_cores=True, bf16="s1"), TF32),            # ZsProb<1, 1, ZO_F32> + ZrProb<0>
         ("tf32", dict(tensor_cores=True), TF32),                          # ZsProb<1, 0, ZO_F32> (|x| in smem) + ZrProb<0>
         ("f16_r", dict(tensor_cores=True, r_f16=True), TF32),             # ZsProb<1, 0, ZO_F16S> + ZrProb<2>
         ("f16_r_s1", dict(tensor_cores=True, bf16="s1", r_f16=True), TF32),   # ZsProb<1, 1, ZO_F16S> + ZrProb<2>
         ("bf16_r", dict(tensor_cores=True, bf16=True), BF16_R),           # ZsProb<1, 0, ZO_BF16> + ZrProb<1>
         ("lrp_tc", dict(variant="lrp_tc"), TF32)]                         # LrpSProb (registers) + LrpRProb
# (rows, in, out): the S kernel reduces over in, the R kernel over out
RULE_SHAPES = [(1, 128, 128), (127, 384, 128), (129, 128, 3072), (129, 3072, 384), (20000, 384, 384)]


@pytest.mark.parametrize("alpha", [1.0, 2.0])
@pytest.mark.parametrize("rows,inf,outf", RULE_SHAPES)
def test_linear_rules(rows, inf, outf, alpha):
    x, w, b, r = inputs(rows + inf + outf, (rows, inf), (outf, inf), (outf,), (rows, outf))
    w *= inf ** -0.5
    r = r.abs()
    xd, wd, bd, rd = x.cuda(), w.cuda(), b.cuda(), r.cuda()
    yd = ops.linear_forward(xd, wd, bd)
    xx, ww, rr = x.double(), w.double(), r.double()
    refs = {False: alphabeta.linear_relprop(xx, ww, rr, alpha=alpha), True: alphabeta.linear_relprop_lrp(xx, ww, rr, alpha=alpha)}
    for name, kw, bound in RULES:
        lrp = kw.get("variant") == "lrp_tc"

        def run(xi, ri, yi, kw=kw, lrp=lrp):
            extra = {} if lrp else dict(y=yi, bias=bd)
            return ops.linear_relprop(xi, wd, ri, alpha=alpha, **kw, **extra)

        try:
            check_rows(run, [xd, rd, yd], refs[lrp], bound)
        except AssertionError as e:
            raise AssertionError("%s: %s" % (name, e)) from None
