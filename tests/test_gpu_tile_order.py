"""The Linear-rule tensor-core GEMMs run their tiles column-fastest (column tile in blockIdx.x) while the m-tiles fit in
gridDim.y, and m-tile-fastest beyond 65535 m-tiles.  Every output row depends on its own input row only, so the first and
last rows of a launch too tall for the column-fastest order must equal, bit for bit, the same rows computed by a short
launch that takes it: each family reaches both orders through the ops API."""
import pytest
import torch

from transformer_explainability_b200 import ops

pytestmark = pytest.mark.gpu

TALL = 65535 * 128 + 1          # one m-tile more than gridDim.y holds
EDGE = 1000


def check_rows(fn, *row_inputs):
    """fn(*row_inputs) on all TALL rows vs on the first / last EDGE rows only."""
    full = fn(*row_inputs)
    torch.cuda.synchronize()
    for sl in (slice(0, EDGE), slice(TALL - EDGE, TALL)):
        part = fn(*(t[sl] for t in row_inputs))
        ref = full[sl]
        assert part.dtype == ref.dtype and torch.equal(part.view(torch.int32), ref.contiguous().view(torch.int32)), sl
    del full


def rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g) * scale


def test_forward_families():
    x = rand(TALL, 64, seed=1)
    w, b = rand(128, 64, seed=2, scale=0.125), rand(128, seed=3, scale=0.1)
    check_rows(lambda xx: ops.linear_forward_epi(xx, w, b, epi="bias", family="f16_split")[0], x)      # LinProb<BIAS, LIN_F16X3>
    check_rows(lambda xx: ops.linear_forward_epi(xx, w, b, epi="bias", family="3xtf32")[0], x)         # LinProb<BIAS, LIN_3XTF32>


def test_backward_families():
    w = rand(64, 128, seed=4, scale=0.125)
    dy = rand(TALL, 64, seed=5)
    check_rows(lambda d: ops.linear_backward_tf32(d, w), dy)                                            # LinProb<STORE, LIN_TF32>
    check_rows(lambda d: ops.linear_backward_epi(d, w, epi="store", family="f16"), dy)                 # LinProb<STORE, LIN_F16>


def test_zplus_rule():
    x = rand(TALL, 128, seed=6)
    w, b = rand(128, 128, seed=7, scale=0.09), rand(128, seed=8, scale=0.1)
    r = rand(TALL, 128, seed=9).abs_()
    y = ops.linear_forward(x, w, b, tensor_cores=True)        # the fp32 SIMT GEMM holds at most 65535 m-tiles
    # ZsProb<single, bf16> + ZrProb<0>, then the fp16 second contraction ZsProb<.., F16S> + ZrProb<2>
    check_rows(lambda xx, rr, yy: ops.linear_relprop(xx, w, rr, tensor_cores=True, y=yy, bias=b, bf16="s1"), x, r, y)
    check_rows(lambda xx, rr, yy: ops.linear_relprop(xx, w, rr, tensor_cores=True, y=yy, bias=b, r_f16=True), x, r, y)
