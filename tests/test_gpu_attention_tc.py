"""GPU: the attention-shaped tensor-core contractions (te_tc_wgmma.cu: NnProb behind te_tc_attention_nn, NkProb behind
te_tc_attention_nk; the diagnostic entry points never fall back to SIMT) against float64 einsum on the same data.

Operands sit in the engines' packed layout: q | k | v inside [batch*N, 3D] (lda = 3D, head h at column h*dh of its third); maps
are [batch, H, N, ld_out] with NP = round_up(N, 4) <= ld_out.  Token counts cover one-row tiles, every tile edge (32, 64, 128,
256), several 128-row tiles with a ragged last one, and the ViT / BERT counts; batch 3 x 12 heads makes a ragged tile of one
sample load the next sample's rows, which must never reach the output.

Error measure: every element against its own scale, |alpha| (|A| |B|^T) for that element (float64), not the tensor maximum.
Bounds carried over from tests/test_gpu_tc.py: 3xTF32 1.5e-8 * K + 2e-6 (K = the reduction length: dh for N x N, N for the
token reduction), single-pass TF32 2e-3.  Measured maxima over all shapes of each test, on one H100 80GB HBM3 at a
400 W power limit:
  N x N STORE   3xTF32 6.2e-7 (dh 32), 7.7e-7 (dh 64); single pass 4.4e-4 (dh 32), 3.2e-4 (dh 64)
  N x N MUL     3xTF32 7.7e-7; single pass 2.9e-4
  N x N SD      1.7e-7 relative to safe_divide(E, Z) of the kernel's own Z
  SOFTMAX       7.5e-5 relative to each probability (scores spread to +-80); row sums within 4.7e-7 of 1
  token reduction STORE  3xTF32 7.5e-7; single pass 8.4e-4 (largest at N = 1, 1.0e-4 at N = 577)
  token reduction MUL    3xTF32 1.1e-6; single pass 8.5e-4
"""
import math

import pytest
import torch

from oracle import rules
from transformer_explainability_b200 import _lib, ops

pytestmark = pytest.mark.gpu

NS = [1, 2, 3, 5, 17, 31, 32, 33, 50, 64, 65, 127, 128, 129, 197, 198, 255, 256, 257, 300, 384, 511, 577]
NS_SAMPLE = [1, 5, 33, 65, 129, 197, 256, 257, 300, 577]      # the other epilogues: every tile-edge class, fewer counts
BH = [(1, 1), (3, 12)]
SENTINEL_ROWS = 2
BOUND_SP = 2e-3
NAN = float("nan")


def f32(a):
    """alpha as the kernel receives it (a C float)"""
    return float(torch.tensor(a, dtype=torch.float32))


def bound_3x(K):
    return 1.5e-8 * K + 2e-6


def npad(n):
    return (n + 3) & ~3


def packed_qkv(batch, heads, n, dh, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(batch * n, 3 * heads * dh, generator=g, device="cuda") * scale


def heads_of(qkv, part, batch, heads, n, dh):
    """[batch, heads, n, dh] float64 view of q (part 0), k (1) or v (2)."""
    D = heads * dh
    return qkv[:, part * D:(part + 1) * D].double().reshape(batch, n, heads, dh).permute(0, 2, 1, 3)


class MapBuf:
    """[batch, heads, n, ld] map in a NaN-filled buffer with sentinel rows after it."""
    def __init__(self, batch, heads, n, ld, fill=NAN):
        self.shape, self.ld, self.np = (batch, heads, n), ld, npad(n)
        self.size = batch * heads * n * ld
        self.buf = torch.full((self.size + SENTINEL_ROWS * ld,), fill, device="cuda")

    @property
    def map(self):
        return self.buf[:self.size].view(*self.shape, self.ld)

    def check_layout(self, what):
        """[.., :N] written (finite), [.., N:NP] exact zeros, [.., NP:ld] and the sentinel rows untouched (NaN)."""
        m, n = self.map, self.shape[2]
        assert torch.isfinite(m[..., :n]).all(), "%s: an element of [.., :N] was not written" % what
        assert (m[..., n:self.np] == 0).all(), "%s: the row padding N..NP-1 is not exact zeros" % what
        assert torch.isnan(m[..., self.np:]).all(), "%s: a column from NP to ld_out was written" % what
        assert torch.isnan(self.buf[self.size:]).all(), "%s: written past the last row" % what


def per_element(out, ref, scale):
    """max |out - ref| / scale over the elements with scale > 0; elements with scale 0 must be exactly ref (0)."""
    out = out.double()
    live = scale > 0
    assert (out[~live] == ref[~live]).all()
    return ((out - ref).abs()[live] / scale[live]).max().item() if live.any() else 0.0


def run_nn(qkv, batch, heads, n, dh, ld, epi, alpha, e=None, single_pass=False, fill=NAN):
    D = heads * dh
    mb = MapBuf(batch, heads, n, ld, fill)
    ops.tc_attention_nn(qkv, 3 * D, qkv[:, D:], 3 * D, batch, heads, n, dh, mb.buf, ld,
                        None if e is None else e.buf, alpha, epi, single_pass)
    return mb


def e_map(batch, heads, n, ld, seed, fn=None):
    """an E operand [batch, heads, n, ld] with NaN in every padding column (the kernels must not let it through)"""
    mb = MapBuf(batch, heads, n, ld)
    g = torch.Generator(device="cuda").manual_seed(seed)
    mb.map[..., :n] = torch.rand(batch, heads, n, n, generator=g, device="cuda") + 0.5 if fn is None else fn
    return mb


@pytest.mark.parametrize("batch,heads", BH)
@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("n", NS)
def test_nn_store(n, dh, batch, heads):
    """out = alpha q k^T, 3xTF32 at every N (and single-pass TF32 at N <= 256, where the engines use it)."""
    qkv = packed_qkv(batch, heads, n, dh, seed=n * 7 + dh + batch)
    q, k = heads_of(qkv, 0, batch, heads, n, dh), heads_of(qkv, 1, batch, heads, n, dh)
    alpha = f32(1.0 / math.sqrt(dh))
    ref = alpha * torch.einsum("bhid,bhjd->bhij", q, k)
    scale = alpha * torch.einsum("bhid,bhjd->bhij", q.abs(), k.abs())
    ld = npad(n) + (8 if batch > 1 else 0)                            # ld_out > NP as well
    for sp in ([False, True] if n <= 256 else [False]):
        mb = run_nn(qkv, batch, heads, n, dh, ld, "store", alpha, single_pass=sp)
        torch.cuda.synchronize()
        mb.check_layout("nn STORE sp=%s" % sp)
        e = per_element(mb.map[..., :n], ref, scale)
        print("nn STORE n %d dh %d batch %d heads %d single_pass %s: %.2e" % (n, dh, batch, heads, sp, e))
        assert e < (BOUND_SP if sp else bound_3x(dh))


@pytest.mark.parametrize("batch,heads", BH)
@pytest.mark.parametrize("n", NS_SAMPLE)
def test_nn_mul(n, batch, heads):
    """out = alpha (dctx v^T) * E (attn_cam = P * (S v^T) / 2): 3xTF32 and, at N <= 256, single pass; NaN in E's padding."""
    dh = 64
    qkv = packed_qkv(batch, heads, n, dh, seed=n * 11 + batch)
    q, k = heads_of(qkv, 0, batch, heads, n, dh), heads_of(qkv, 1, batch, heads, n, dh)
    ld = npad(n) + 4
    e = e_map(batch, heads, n, ld, seed=n)
    E = e.map[..., :n].double()
    alpha = 0.5
    ref = alpha * torch.einsum("bhid,bhjd->bhij", q, k) * E
    scale = alpha * torch.einsum("bhid,bhjd->bhij", q.abs(), k.abs()) * E.abs()
    for sp in ([False, True] if n <= 256 else [False]):
        mb = run_nn(qkv, batch, heads, n, dh, ld, "mul", alpha, e=e, single_pass=sp)
        torch.cuda.synchronize()
        mb.check_layout("nn MUL sp=%s" % sp)
        err = per_element(mb.map[..., :n], ref, scale)
        print("nn MUL n %d batch %d heads %d single_pass %s: %.2e" % (n, batch, heads, sp, err))
        assert err < (BOUND_SP if sp else bound_3x(dh))


@pytest.mark.parametrize("batch,heads", BH)
@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("n", [1, 5, 33, 129, 257, 577])
def test_nn_sd(n, dh, batch, heads):
    """out = safe_divide(E, alpha q k^T) (the matmul1 rule's S1).  E = Z^2 u keeps S = Z u continuous through Z = 0
    (test_gpu_rules.py::test_attention_matmul_rules); zeroed q rows make Z exactly 0 on the tensor cores too, where the
    result must be exactly 0 (te_sd_fast).  The epilogue is checked against safe_divide of the kernel's own Z (STORE output,
    same accumulation): te_sd_fast divides with rcp.approx, 2 ulp, so 4e-7 relative."""
    qkv = packed_qkv(batch, heads, n, dh, seed=n * 13 + dh + batch)
    zero_rows = list(range(0, batch * n, 7))
    qkv[zero_rows, :heads * dh] = 0.0
    q, k = heads_of(qkv, 0, batch, heads, n, dh), heads_of(qkv, 1, batch, heads, n, dh)
    alpha = f32(1.0 / math.sqrt(dh))
    ld = npad(n)
    z64 = alpha * torch.einsum("bhid,bhjd->bhij", q, k)
    g = torch.Generator(device="cuda").manual_seed(n + 1)
    e = e_map(batch, heads, n, ld, seed=0, fn=(z64 ** 2 * torch.rand(z64.shape, generator=g, device="cuda", dtype=torch.float64)).float())
    zk = run_nn(qkv, batch, heads, n, dh, ld, "store", alpha)
    mb = run_nn(qkv, batch, heads, n, dh, ld, "sd", alpha, e=e)
    torch.cuda.synchronize()
    mb.check_layout("nn SD")
    out = mb.map[..., :n].double()
    ref = rules.safe_divide(e.map[..., :n].double(), zk.map[..., :n].double())
    err = ((out - ref).abs() / ref.abs().clamp_min(1e-300)).max().item()
    print("nn SD n %d dh %d batch %d heads %d: %.2e relative to safe_divide(E, Z_kernel)" % (n, dh, batch, heads, err))
    assert err < 4e-7
    zero = torch.zeros(batch * n, dtype=torch.bool, device="cuda")
    zero[zero_rows] = True
    zero = zero.view(batch, n)[:, None, :, None].expand(batch, heads, n, n)
    assert (zk.map[..., :n][zero] == 0).all() and (out[zero] == 0).all(), "an exactly-zero Z did not give exactly 0"


@pytest.mark.parametrize("batch,heads", BH)
@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("n", [1, 2, 5, 31, 33, 64, 65, 127, 129, 197, 255, 256])
def test_nn_softmax(n, dh, batch, heads):
    """P = softmax(alpha q k^T) over the keys, fused in the epilogue (N <= 256), scores spread to +-80 so that the row-max
    subtraction matters.  A score error d perturbs every probability by at most 2 |d| relative: with the 3xTF32 bound on
    the scores and the 2^-22 of ex2.approx, the stated per-element bound is 2 alpha max_j(|q||k|^T) * bound_3x(dh) + 1e-5,
    relative to each probability (> 1e-30; ex2.approx.ftz flushes below 2^-126).  Rows sum to 1 within 1e-6."""
    qkv = packed_qkv(batch, heads, n, dh, seed=n * 17 + dh + batch)
    q, k = heads_of(qkv, 0, batch, heads, n, dh), heads_of(qkv, 1, batch, heads, n, dh)
    s64 = torch.einsum("bhid,bhjd->bhij", q, k)
    alpha = f32(80.0 / s64.abs().max().item())
    ref = torch.softmax(alpha * s64, dim=-1)
    rowscale = alpha * torch.einsum("bhid,bhjd->bhij", q.abs(), k.abs()).amax(dim=-1, keepdim=True)
    ld = npad(n) + (4 if batch > 1 else 0)
    mb = run_nn(qkv, batch, heads, n, dh, ld, "softmax", alpha)
    torch.cuda.synchronize()
    mb.check_layout("nn SOFTMAX")
    p = mb.map[..., :n].double()
    live = ref > 1e-30
    relerr = ((p - ref).abs() / ref.clamp_min(1e-300))[live]
    bound = (2 * rowscale * bound_3x(dh) + 1e-5).expand_as(ref)[live]
    print("nn SOFTMAX n %d dh %d batch %d heads %d: max rel %.2e (bound %.1e), row sums %.2e" % (
        n, dh, batch, heads, relerr.max().item(), bound.min().item(), (p.sum(-1) - 1).abs().max().item()))
    assert (relerr < bound).all()
    assert ((p - ref).abs()[~live] < 1e-30).all()
    assert (p.sum(-1) - 1).abs().max().item() < 1e-6


def _status(fn, *args, **kw):
    try:
        fn(*args, **kw)
    except _lib.TeError as e:
        return e.status
    return 0


def test_nn_nk_unsupported_shapes_do_not_run():
    """Shapes the tensor-core kernels do not take return TE_ERR_UNSUPPORTED and leave out untouched: dh not in {32, 64},
    NP % 4 != 0 (token reduction), the fused softmax beyond one 256-key tile, the single-pass kernel with SD / SOFTMAX."""
    U = _lib.TE_ERR_UNSUPPORTED
    for dh in (16, 48, 128):
        qkv = packed_qkv(1, 2, 40, dh, seed=dh)
        mb = MapBuf(1, 2, 40, 40)
        assert _status(ops.tc_attention_nn, qkv, 6 * dh, qkv[:, 2 * dh:], 6 * dh, 1, 2, 40, dh, mb.buf, 40) == U
        assert torch.isnan(mb.buf).all()
    qkv = packed_qkv(1, 1, 257, 64, seed=257)
    mb = MapBuf(1, 1, 257, 260)
    assert _status(ops.tc_attention_nn, qkv, 192, qkv[:, 64:], 192, 1, 1, 257, 64, mb.buf, 260, epi="softmax") == U
    e = e_map(1, 1, 257, 260, seed=1)
    assert _status(ops.tc_attention_nn, qkv, 192, qkv[:, 64:], 192, 1, 1, 257, 64, mb.buf, 260, e=e.buf, epi="sd",
                   single_pass=True) == U
    assert torch.isnan(mb.buf).all()
    # ragged lda: not a multiple of 4
    x = torch.randn(64 * 67, device="cuda")
    assert _status(ops.tc_attention_nn, x, 67, x, 67, 1, 1, 64, 64, mb.buf, 64) == U
    amap = torch.rand(1, 1, 33, 34, device="cuda")
    out = torch.full((33, 64), NAN, device="cuda")
    assert _status(ops.tc_attention_nk, amap, 34, 0, qkv, 192, 1, 1, 33, out, 64) == U
    assert torch.isnan(out).all()
    assert _lib.TE_ERR_UNSUPPORTED == -4


# ---- token reduction: out[b*N+m, h*64+d] = alpha sum_k M_h[m,k] X[b*N+k, h*64+d] -----------------------------------------------
def nk_case(n, batch, heads, seed, epi):
    dh, D = 64, heads * 64
    qkv = packed_qkv(batch, heads, n, dh, seed=seed)
    np_ = npad(n)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    amap = torch.full((batch, heads, n, np_), NAN, device="cuda")         # the padding columns are never read
    amap[..., :n] = torch.randn(batch, heads, n, n, generator=g, device="cuda")
    ld_out = D + 8
    E = None
    if epi == "mul":
        E = torch.full((batch * n + SENTINEL_ROWS, ld_out), NAN, device="cuda")
        E[:batch * n, :D] = torch.rand(batch * n, D, generator=g, device="cuda") + 0.5
    return qkv, amap, np_, ld_out, E


@pytest.mark.parametrize("batch,heads", BH)
@pytest.mark.parametrize("amn", [0, 1])
@pytest.mark.parametrize("n", NS)
def test_nk_store(n, amn, batch, heads):
    """out = alpha M v (amn 0: attn v, dS k, S1 k) or alpha M^T v (amn 1: attn^T dctx, dS^T q, S1^T q), 3xTF32 and single
    pass, with NaN in the map's padding columns; the columns of out beyond heads * 64 and the rows after it stay untouched."""
    D = heads * 64
    alpha = 0.75
    qkv, amap, np_, ld_out, _ = nk_case(n, batch, heads, seed=n * 19 + amn + batch, epi="store")
    m = amap[..., :n].double()
    if amn:
        m = m.transpose(-1, -2)
    v = heads_of(qkv, 2, batch, heads, n, 64)
    ref = (alpha * m @ v).permute(0, 2, 1, 3).reshape(batch * n, D)
    scale = (alpha * m.abs() @ v.abs()).permute(0, 2, 1, 3).reshape(batch * n, D)
    for sp in (False, True):
        out = torch.full((batch * n + SENTINEL_ROWS, ld_out), NAN, device="cuda")
        ops.tc_attention_nk(amap, np_, amn, qkv[:, 2 * D:], 3 * D, batch, heads, n, out, ld_out, None, alpha, "store", sp)
        torch.cuda.synchronize()
        assert torch.isfinite(out[:batch * n, :D]).all(), "an element was not written (or padding leaked in)"
        assert torch.isnan(out[:batch * n, D:]).all() and torch.isnan(out[batch * n:]).all(), "written outside the output"
        e = per_element(out[:batch * n, :D], ref, scale)
        print("nk STORE n %d amn %d batch %d heads %d single_pass %s: %.2e" % (n, amn, batch, heads, sp, e))
        assert e < (BOUND_SP if sp else bound_3x(n))


@pytest.mark.parametrize("batch,heads", BH)
@pytest.mark.parametrize("amn", [0, 1])
@pytest.mark.parametrize("n", NS_SAMPLE)
def test_nk_mul(n, amn, batch, heads):
    """out = alpha (M v) * E (R_v = v * (P^T S) / 2, R_q = q * (S1 k) / 2 ...), NaN in the map's and E's padding."""
    D = heads * 64
    alpha = 0.5
    qkv, amap, np_, ld_out, E = nk_case(n, batch, heads, seed=n * 23 + amn + batch, epi="mul")
    m = amap[..., :n].double()
    if amn:
        m = m.transpose(-1, -2)
    v = heads_of(qkv, 2, batch, heads, n, 64)
    e64 = E[:batch * n, :D].double()
    ref = (alpha * m @ v).permute(0, 2, 1, 3).reshape(batch * n, D) * e64
    scale = (alpha * m.abs() @ v.abs()).permute(0, 2, 1, 3).reshape(batch * n, D) * e64
    for sp in (False, True):
        out = torch.full((batch * n + SENTINEL_ROWS, ld_out), NAN, device="cuda")
        ops.tc_attention_nk(amap, np_, amn, qkv[:, 2 * D:], 3 * D, batch, heads, n, out, ld_out, E, alpha, "mul", sp)
        torch.cuda.synchronize()
        assert torch.isfinite(out[:batch * n, :D]).all()
        assert torch.isnan(out[:batch * n, D:]).all() and torch.isnan(out[batch * n:]).all()
        e = per_element(out[:batch * n, :D], ref, scale)
        print("nk MUL n %d amn %d batch %d heads %d single_pass %s: %.2e" % (n, amn, batch, heads, sp, e))
        assert e < (BOUND_SP if sp else bound_3x(n))
