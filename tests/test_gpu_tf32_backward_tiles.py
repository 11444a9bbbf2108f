"""GPU: the single-pass TF32 backward Linear (STORE) on 256-column tiles.

Its column tiles are 256 wide, so at N = 128 (mod 256) the last tile covers 128 columns past the output.  At such shapes,
with M not a multiple of the 128-row tile, dx = dy W must stay within the fp64 bound of tests/test_gpu_tc.py (2e-3 of the
tensor maximum) and the kernel must write nothing past the output.
"""
import pytest
import torch

from transformer_explainability_b200 import _lib, ops
from transformer_explainability_b200._lib import check, ptr

pytestmark = pytest.mark.gpu

TF32 = _lib.FLAG_LINEAR_TENSOR_CORES | _lib.FLAG_BACKWARD_TF32


def _backward(dy, w, dx, scratch):
    """dx = dy W on the single-pass TF32 kernel (STORE) into dx's storage (row stride in_features)"""
    check(_lib.load().te_linear_backward(ptr(dy), ptr(w), None, ptr(dx), ptr(scratch), dy.shape[0], w.shape[1], w.shape[0],
                                         ops.LINEAR_EPI["store"], TF32,
                                         _lib.ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "te_linear_backward")


@pytest.mark.parametrize("rows,inf,outf", [(333, 384, 256), (200, 640, 768), (129, 128, 384)])
def test_tf32_backward_partial_column_tile(rows, inf, outf):
    g = torch.Generator().manual_seed(rows * 7 + inf)
    w = torch.randn(outf, inf, generator=g) * 0.05
    dy = torch.randn(rows, outf, generator=g)
    wd, dyd = w.cuda(), dy.cuda()
    pad = 3 * inf + 5                                 # floats behind the output: poisoned, must stay so
    buf = torch.full((rows * inf + pad,), float("nan"), device="cuda")
    scratch = torch.empty(16 * w.numel(), device="cuda")
    _backward(dyd, wd, buf, scratch)
    torch.cuda.synchronize()
    out = buf[:rows * inf].view(rows, inf).double().cpu()
    ref = dy.double() @ w.double()
    e = ((out - ref).abs().max() / ref.abs().max()).item()
    print("tf32 backward rows %d in %d out %d: rel %.2e" % (rows, inf, outf, e))
    assert e < 2e-3
    assert torch.isnan(buf[rows * inf:]).all(), "the kernel wrote past the output"
    assert torch.equal(ops.linear_backward_tf32(dyd, wd).cpu(), out.float())
