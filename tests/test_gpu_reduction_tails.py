"""GPU: the chunked Linear GEMMs on reductions that end in a partial chunk, against fp64.

The 3xTF32 and fp16 forms of ``wg_kernel`` (``LinProb`` in te_tc_wgmma.cu) fold their accumulators into the running total
once per 128 elements of the reduction: 3xTF32 every four 32-wide k-blocks, the fp16 forms (forward split, single-pass
backward) every two 64-wide k-blocks, each fold times the A operand's block scale of that chunk (``LinProb::chunk_scale``,
``rs_ld = ceil(K / 128)`` scales per row).  A reduction of K = 128 c + 64 (192: the ViT-Ti fc1 forward and fc2 backward;
320; 576) runs c full chunks and then a half one, which folds on the ``it + 1 == kb`` branch with the scale of a half-filled
block.  K = 32 and 96 are one partial chunk only.  N = 128 is one column tile, 384 / 640 are N % 256 == 128.

Stress data: row magnitudes over six decades, and the columns of the last 128-wide block of A scaled by 2^20 in the even
rows and by 2^-20 in the odd rows.  That block's fp16 scale is then 2^-+20 times block 0's: a fold with the wrong scale
column is a 2^20 error, a dropped or doubled last fold an O(1) error of the even rows.

Bounds per element, relative to the element's own scale |A||B|^T (+ |bias|), and the GELU epilogue bounds: those of
tests/test_gpu_tc.py (LIN_BOUND).  The producers of the fp16 operand format at these widths (``te_f16_block_split``,
``te_layernorm_split``) are bit-exact against oracle/f16_split.split_rows, scale array [rows, ceil(cols / 128)] included.
"""
import numpy as np
import pytest
import torch

from oracle import f16_split as F
from test_gpu_tc import GELU_GRAD_EXACT, GELU_GRAD_FAST, LIN_BOUND, _e0_grid, _gelu64, _gelu_grad64, elem_err
from transformer_explainability_b200 import ops

pytestmark = pytest.mark.gpu

TAIL = 2.0 ** 20


def tail_stress(a):
    """scale the last 128-column block of a [rows, K] by 2^20 in the even rows and 2^-20 in the odd rows (in place)"""
    last = (a.shape[1] - 1) // 128 * 128
    a[0::2, last:] *= TAIL
    a[1::2, last:] /= TAIL
    return a


@pytest.mark.parametrize("K", [32, 96, 192, 320, 576])
@pytest.mark.parametrize("rows", [1, 65, 591])
def test_linear_forward_partial_last_chunk(rows, K):
    g = torch.Generator(device="cuda").manual_seed(rows * 7 + K)
    x = torch.randn(rows, K, generator=g, device="cuda") * torch.logspace(-3, 3, rows, device="cuda")[:, None]
    tail_stress(x)
    for N in (128, 384, 640):
        w = torch.randn(N, K, generator=g, device="cuda") * 0.05
        b = torch.randn(N, generator=g, device="cuda") * 0.1
        e0 = torch.randn(rows, N, generator=g, device="cuda")
        xw = x.double() @ w.double().T
        sxw = x.double().abs() @ w.double().abs().T
        for family in ("simt", "3xtf32", "f16_split"):
            if family == "f16_split" and K % 64:
                continue
            bound = LIN_BOUND[family](K)
            for epi in ("store", "bias", "bias_gelu", "bias_add"):
                biased = epi != "store"
                y64 = xw + b.double() if biased else xw
                scale = sxw + b.double().abs() if biased else sxw
                y, y2 = ops.linear_forward_epi(x, w, b if biased else None, e0 if epi == "bias_add" else None, epi=epi,
                                               family=family)
                torch.cuda.synchronize()
                ey = elem_err(y, y64, scale)
                e2, b2 = 0.0, 1.0
                if epi == "bias_gelu":          # |GELU'| <= 1.13, plus the fp32 GELU itself
                    e2, b2 = elem_err(y2, _gelu64(y64), 1.13 * scale), bound + 5e-7
                elif epi == "bias_add":         # e0 + y in fp32: one rounding of |e0| + |y|
                    e2, b2 = elem_err(y2, e0.double() + y64, scale + e0.double().abs()), bound + 1.2e-7
                print("fwd %s %s rows %d K %d N %d: y %.2e y2 %.2e (bound %.1e)" % (family, epi, rows, K, N, ey, e2, bound))
                assert ey < bound and e2 < b2, (family, epi, N)


@pytest.mark.parametrize("K", [192, 320, 576])
@pytest.mark.parametrize("rows", [1, 65, 591])
def test_linear_backward_partial_last_chunk(rows, K):
    """dx = dy W (reduction over the Linear's out = K), STORE and GELU_BWD; the GELU_BWD measure is that of
    test_gpu_tc.py::test_linear_backward_gelu_epilogue"""
    g = torch.Generator(device="cuda").manual_seed(rows * 11 + K)
    dy = torch.randn(rows, K, generator=g, device="cuda") * torch.logspace(-3, 3, rows, device="cuda")[:, None]
    tail_stress(dy)
    for N in (128, 384):
        w = torch.randn(K, N, generator=g, device="cuda") * 0.05
        e0 = _e0_grid(rows, N, g)
        gp = _gelu_grad64(e0.double())
        v64 = dy.double() @ w.double()
        scale = dy.double().abs() @ w.double().abs()
        for family in ("simt", "3xtf32", "tf32", "f16"):
            bound = LIN_BOUND[family](K)
            gb = GELU_GRAD_FAST if family == "tf32" else GELU_GRAD_EXACT
            v = ops.linear_backward_epi(dy, w, None, epi="store", family=family)
            dx = ops.linear_backward_epi(dy, w, e0, epi="gelu_bwd", family=family)
            torch.cuda.synchronize()
            ev = elem_err(v, v64, scale)
            eg = elem_err(dx, v64 * gp, scale * ((bound + 1.2e-7) * gp.abs() + gb))
            print("bwd %s rows %d K %d N %d: store %.2e (bound %.1e), gelu_bwd %.2f of its bound" % (
                family, rows, K, N, ev, bound, eg))
            assert ev < bound and eg < 1, (family, N)


@pytest.mark.parametrize("cols", [64, 192, 320, 576])
def test_f16_block_split_partial_block_bit_exact(cols):
    g = torch.Generator().manual_seed(cols)
    rows = 300
    x = torch.randn(rows, cols, generator=g) * torch.logspace(-3, 1, cols)
    x = tail_stress(x * torch.logspace(-20, 20, rows)[:, None])     # rows over 40 decades, all of them normal fp32
    x[7] = 0.0
    hi, lo, si = ops.f16_block_split(x.cuda())
    torch.cuda.synchronize()
    rh, rl, rs = F.split_rows(x.numpy())
    assert si.shape == (rows, -(-cols // 128))
    assert np.array_equal(si.cpu().numpy(), rs)
    assert np.array_equal(hi.cpu().numpy().view(np.uint16), rh.view(np.uint16))
    assert np.array_equal(lo.cpu().numpy().view(np.uint16), rl.view(np.uint16))


@pytest.mark.parametrize("D", [192, 320])
def test_layernorm_split_partial_block_bit_exact(D):
    """the split of the kernel's own y; the LayerNorm weight spans 60 decades and lifts the last block by 2^20"""
    g = torch.Generator().manual_seed(D)
    rows = 300
    x = torch.randn(rows, D, generator=g) * torch.logspace(-3, 1, D) + torch.randn(rows, 1, generator=g)
    x[7] = 0.0
    w = torch.randn(D, generator=g) * torch.logspace(-30, 30, D)
    w[(D - 1) // 128 * 128:] *= TAIL
    y, _, _, hi, lo, si = ops.layernorm_split(x.cuda(), w.cuda(), torch.zeros(D).cuda(), 1e-6)
    torch.cuda.synchronize()
    rh, rl, rs = F.split_rows(y.cpu().numpy())
    assert si.shape == (rows, -(-D // 128))
    assert np.array_equal(si.cpu().numpy(), rs)
    assert np.array_equal(hi.cpu().numpy().view(np.uint16), rh.view(np.uint16))
    assert np.array_equal(lo.cpu().numpy().view(np.uint16), rl.view(np.uint16))
    assert (si.cpu()[7] == 1).all() and (hi.cpu()[7] == 0).all()
