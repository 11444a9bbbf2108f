"""GPU: the head reductions, the GradCAM head weights and the heatmap up-sampling against fp64 torch on the same fp32 inputs.

``ops.head_reduce`` (every secondary method: attention / rollout / GradCAM baselines of ViT and BERT),
``ops.head_region_mean`` (the GradCAM head weights) and ``visualization.relevance_to_heatmap`` (the results file of
generate_visualizations, the perturbation and the segmentation evaluation) at the shapes where their kernels can go wrong:
N around a warp (31, 32, 33) and around the model widths (197 ViT, 198 DeiT-distilled, 257, 577 ViT at 384), row strides
N, round_up(N, 4) and round_up(N, 4) + 4 with NaN in every pad column, 1 to 16 heads, and for the heatmap the grids of
ViT-B/32 and ViT-B/16 at 224 and 384 at power-of-two and other scales.

Bounds (u = 2^-24, the unit roundoff of fp32):

- head_reduce, per element, relative to its own scale S = mean_h |a g w|: (H + 3) u S + u |ref|.  The kernel makes at most
  two multiplies per head (a g, then w), H - 1 sequential adds and the division by H, then relu, which is exact.  The other
  relu placement on the same data (mean_relu against the relu_mean reference) must break the bound: sample 0 has one
  positive and one negative head product at element (0, 0), where the two placements differ by at least 1 / H of them.
- head_region_mean: the kernel sums in fp64 and rounds the fp64 mean once, so |out - ref| <= u |ref| + 2 n 2^-53 mean |g|
  over the n elements of the region (the fp64 summation errors of the kernel and of torch): one rounding.
- relevance_to_heatmap: see ``heatmap_bound``.

An empty or out-of-range region of head_region_mean returns TE_ERR_ARG without launching anything.  Mis-shaped operands of
head_reduce and relevance_to_heatmap raise ValueError before the C library is called.
"""
import pytest
import torch
import torch.nn.functional as F

from transformer_explainability_b200 import _lib, ops, visualization

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TE_ERR_ARG = -1                      # include/te_b200.h
NS = [1, 2, 31, 32, 33, 197, 198, 257, 577]
HS = [1, 3, 12, 16]
BS = [1, 3]
LDS = ["n", "np", "np4"]
MODES = ("mean", "relu_mean", "mean_relu")


def _ld(n, kind):
    np_ = (n + 3) // 4 * 4
    return {"n": n, "np": np_, "np4": np_ + 4}[kind]


def _attn(B, H, n, ld, gen):
    """signed [B,H,n,n] view of a [B,H,n,ld] buffer whose pad columns [n, ld) hold NaN"""
    buf = torch.randn(B, H, n, ld, generator=gen, device="cuda")
    buf[..., n:] = float("nan")
    return buf[..., :n]


def _operands(B, H, n, ld, seed, ld_g=None):
    """a, g [B,H,n,n] (row strides ld, ld_g) and head weights [B,H], all signed; with H > 1 the products a g w of sample 0
    at element (0, 0) are positive in head 0 and negative in head 1 (the near miss of the relu placements)"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    a = _attn(B, H, n, ld, gen)
    g = _attn(B, H, n, ld if ld_g is None else ld_g, gen)
    w = torch.randn(B, H, generator=gen, device="cuda")
    if H > 1:
        a[0, 0, 0, 0] = a[0, 0, 0, 0].abs() + 0.5
        a[0, 1, 0, 0] = -(a[0, 1, 0, 0].abs() + 0.5)
        g[0, :2, 0, 0] = g[0, :2, 0, 0].abs() + 0.5
        w[0, :2] = w[0, :2].abs() + 0.5
    return a, g, w


def _head_reduce64(p, mode):
    """the reference's head reductions of the products p [B,H,N,N] (fp64)"""
    if mode == "relu_mean":
        return p.clamp(min=0).mean(1)
    r = p.mean(1)
    return r.clamp(min=0) if mode == "mean_relu" else r


def _ratio(err, bound):
    """max of err / bound; an element whose bound is 0 (every head product exactly 0) must be exact"""
    return (err / bound.clamp(min=1e-300)).max().item()


def check_head_reduce(a, g, w, what):
    """every mode x {g, no g} x {head weights, none} against fp64; returns the largest error / bound"""
    B, H, n, _ = a.shape
    worst = 0.0
    for with_g in (False, True):
        for with_w in (False, True):
            gg, ww = (g if with_g else None), (w if with_w else None)
            p = a.double()
            if with_g:
                p = p * g.double()
            if with_w:
                p = p * w.double()[:, :, None, None]
            scale = p.abs().mean(1)
            res = {}
            for mode in MODES:
                out = ops.head_reduce(a, gg, ww, mode=mode)
                ref = _head_reduce64(p, mode)
                bound = (H + 3) * U * scale + U * ref.abs()
                assert out.shape == (B, n, n) and out.is_contiguous() and out.dtype == torch.float32, what
                assert not torch.isnan(out).any(), (what, mode, with_g, with_w)
                r = _ratio((out.double() - ref).abs(), bound)
                assert r <= 1.0, (what, mode, with_g, with_w, r)
                worst = max(worst, r)
                res[mode] = (out, ref, bound)
            if H > 1:                  # the bound tells the two relu placements apart
                miss = _ratio((res["mean_relu"][0].double() - res["relu_mean"][1]).abs(), res["relu_mean"][2])
                assert miss > 1.0, (what, with_g, with_w, miss)
    return worst


@pytest.mark.parametrize("ld_kind", LDS)
@pytest.mark.parametrize("n", NS)
def test_head_reduce_against_fp64(n, ld_kind):
    ld = _ld(n, ld_kind)
    for H in HS:
        for B in BS:
            a, g, w = _operands(B, H, n, ld, seed=n * 131 + ld * 7 + H * 3 + B)
            e = check_head_reduce(a, g, w, "n %d ld %d H %d B %d" % (n, ld, H, B))
            print("head_reduce n %d ld %d H %d B %d: max err / bound %.3f" % (n, ld, H, B, e))


@pytest.mark.parametrize("n", NS)
def test_head_reduce_operands_of_different_row_strides(n):
    """a with row stride round_up(n, 4) and g with round_up(n, 4) + 4: ops.head_reduce copies both to stride n"""
    ld = _ld(n, "np")
    for H in (3, 12):
        a, g, w = _operands(3, H, n, ld, seed=n * 17 + H, ld_g=ld + 4)
        assert a.stride(2) != g.stride(2)
        e = check_head_reduce(a, g, w, "n %d lds %d / %d H %d" % (n, ld, ld + 4, H))
        print("head_reduce n %d ld a %d g %d H %d B 3: max err / bound %.3f" % (n, ld, ld + 4, H, e))


def test_head_reduce_many_rows():
    """B N = 9232 rows, one warp each: more warps than the 132 SMs of an H100 hold at once (132 x 64 = 8448)"""
    n = 577
    a, g, w = _operands(16, 12, n, _ld(n, "np4"), seed=99)
    e = check_head_reduce(a, g, w, "B 16 n 577 H 12")
    print("head_reduce n 577 H 12 B 16: max err / bound %.3f" % e)


# ---- head_region_mean ----------------------------------------------------------------------------------------------------
def _regions(n):
    """(name, rows, cols) of the regions the GradCAM baselines read, and the edges of the kernel's flat index"""
    c0 = min(3, n - 1)
    c1 = n - 1 if (n - c0) % 32 == 0 and n - c0 > 1 else n
    out = [("whole", None, None),
           ("single", (n // 3, n // 3 + 1), (2 * n // 3, 2 * n // 3 + 1)),
           ("last row", (n - 1, n), (0, n)),
           ("last column", (0, n), (n - 1, n)),
           ("ragged", (n // 4, n - n // 5), (c0, c1))]
    if n >= 2:
        out.append(("vit", (0, 1), (1, n)))
    if n >= 3:
        out.append(("deit", (0, 1), (2, n)))
    return out


@pytest.mark.parametrize("ld_kind", LDS)
@pytest.mark.parametrize("n", NS)
def test_head_region_mean_against_fp64(n, ld_kind):
    ld = _ld(n, ld_kind)
    worst = 0.0
    for H in HS:
        for B in BS:
            g = _attn(B, H, n, ld, torch.Generator(device="cuda").manual_seed(n * 7 + ld + H * 5 + B))
            g += 0.25                                          # a mean that does not cancel; the pads stay NaN
            for name, rows, cols in _regions(n):
                r0, r1 = rows if rows is not None else (0, n)
                c0, c1 = cols if cols is not None else (0, n)
                out = ops.head_region_mean(g, rows, cols)
                reg = g.double()[:, :, r0:r1, c0:c1]
                ref = reg.mean(dim=(2, 3))
                bound = U * ref.abs() + 2 * reg[0, 0].numel() * 2.0 ** -53 * reg.abs().mean(dim=(2, 3))
                assert out.shape == (B, H) and not torch.isnan(out).any(), (n, ld, H, B, name)
                r = ((out.double() - ref).abs() / bound).max().item()
                assert r <= 1.0, (n, ld, H, B, name, r)
                worst = max(worst, r)
    print("head_region_mean n %d ld %d: max err / bound %.3f" % (n, ld, worst))


@pytest.mark.parametrize("rows,cols", [((5, 5), None), ((6, 5), None), ((0, 34), None), ((-1, 3), None),
                                       (None, (7, 7)), (None, (9, 2)), (None, (0, 34)), (None, (-2, 4))])
def test_head_region_mean_refuses_bad_regions(rows, cols):
    """n = 33: an empty region, one past the map or one with a negative start is TE_ERR_ARG, and nothing is written"""
    n = 33
    g = _attn(2, 3, n, _ld(n, "np"), torch.Generator(device="cuda").manual_seed(4))
    with pytest.raises(_lib.TeError) as err:
        ops.head_region_mean(g, rows, cols)
    assert err.value.status == TE_ERR_ARG
    r0, r1 = rows if rows is not None else (0, n)
    c0, c1 = cols if cols is not None else (0, n)
    out = torch.full((2, 3), 7.0, device="cuda")
    st = _lib.load().te_head_region_mean(_lib.ptr(g), 2, 3, n, g.stride(2), r0, r1, c0, c1, _lib.ptr(out),
                                         _lib.ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert st == TE_ERR_ARG and bool((out == 7.0).all())


# ---- relevance_to_heatmap ------------------------------------------------------------------------------------------------
def heatmap64(maps, grid, scale):
    """example.ipynb:57-60 in fp64: bilinear x scale (align_corners=False), then the per-sample min-max"""
    t = F.interpolate(maps.double().reshape(-1, 1, grid, grid), scale_factor=scale, mode="bilinear")
    t = t.reshape(maps.shape[0], -1)
    lo, hi = t.amin(1, keepdim=True), t.amax(1, keepdim=True)
    return ((t - lo) / (hi - lo)).reshape(-1, grid * scale, grid * scale), (hi - lo).reshape(-1)


def heatmap_bound(maps, grid, scale, rng):
    """Per-sample bound on |kernel - fp64| for finite maps, M = max |m| of the sample, R = the fp64 range of its up-sampled map.

    Up-sampled value v = ly0 (lx0 a + lx1 b) + ly1 (lx0 c + lx1 d) in fp32:
      - three roundings in each inner sum and three in the outer one, each at most u M: 6 u M;
      - lx0 = 1 - lx1 and ly0 = 1 - ly1 round by at most u / 2 each: u M;
      - the source coordinate s = 1/scale (y + 0.5) - 0.5 is exact for a power-of-two scale.  Otherwise 1/scale, the
        product and the subtraction each round by at most u grid, and v is 2M-Lipschitz in s (bilinear
        interpolation is continuous across the cell edges and the clamps), so the x and y coordinates add 12 u grid M.
    So |v - v64| <= eps = (7 + 12 grid [scale not a power of two]) u M.  The min and the max move by eps each, so v - min
    and the range by 2 eps each; with (v - min) / range <= 1 and three more roundings (subtraction, range, division) the
    normalised pixel is off by at most 4 eps / R + 3 u (4 u here, for the second-order terms)."""
    pow2 = scale & (scale - 1) == 0
    eps = (7 + (0 if pow2 else 12 * grid)) * U * maps.double().abs().amax(1)
    return 4 * eps / rng + 4 * U


def _maps(B, grid, seed):
    """signed maps, sample b scaled by 10^-b and offset by b of its scale (a range well below max |m|)"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    b = torch.arange(B, device="cuda", dtype=torch.float32)[:, None]
    return (torch.randn(B, grid * grid, generator=gen, device="cuda") + b) * 10.0 ** -b


@pytest.mark.parametrize("B", [1, 5])
@pytest.mark.parametrize("scale", [3, 12, 16, 32])
@pytest.mark.parametrize("grid", [7, 14, 24])
def test_heatmap_against_fp64(grid, scale, B):
    G = grid * scale
    maps = _maps(B, grid, seed=grid * 100 + scale * 10 + B)
    heat = visualization.relevance_to_heatmap(maps, grid=grid, scale=scale)
    ref, rng = heatmap64(maps, grid, scale)
    bound = heatmap_bound(maps, grid, scale, rng)
    assert heat.shape == (B, G, G) and heat.is_cuda and heat.is_contiguous()
    err = (heat.double() - ref).abs().reshape(B, -1).amax(1)
    print("heatmap grid %d scale %d B %d: max err %s, bound %s" % (
        grid, scale, B, ["%.2e" % e for e in err.tolist()], ["%.2e" % e for e in bound.tolist()]))
    assert bool((err <= bound).all()), (err, bound)
    flat = heat.reshape(B, -1)
    assert bool((flat.amin(1) == 0).all() and (flat.amax(1) == 1).all())        # (max - min) / (max - min) is exactly 1

    # a constant map normalises to 0 / 0 = NaN everywhere, as in torch.  The constants are chosen so that the interpolated
    # map is exactly constant in fp32 too (zero or a power of two: every product with a weight is exact and the weights of
    # each axis round to a sum of exactly 1)
    for c in (0.0, 2.0 ** -12, -1.0):
        const = torch.full((B, grid * grid), c, device="cuda")
        assert bool(torch.isnan(visualization.relevance_to_heatmap(const, grid=grid, scale=scale)).all()), c
        assert bool(torch.isnan(heatmap64(const, grid, scale)[0]).all()), c

    # one NaN in one sample: that sample is NaN everywhere, as torch's min / max make it; the others are unchanged
    k = B // 2
    nan_maps = maps.clone()
    nan_maps[k, (grid * grid) // 3] = float("nan")
    nheat = visualization.relevance_to_heatmap(nan_maps, grid=grid, scale=scale)
    assert bool(torch.isnan(heatmap64(nan_maps, grid, scale)[0][k]).all())
    assert bool(torch.isnan(nheat[k]).all()), "%d of %d pixels NaN" % (int(torch.isnan(nheat[k]).sum()), G * G)
    others = [b for b in range(B) if b != k]
    assert torch.equal(nheat[others], heat[others])


# ---- operand checks before any launch -------------------------------------------------------------------------------------
@pytest.fixture
def no_launch(monkeypatch):
    """the C library may not be reached: any call into it fails the test"""
    def refuse():
        raise AssertionError("the C library was called")
    monkeypatch.setattr(_lib, "load", refuse)


def test_head_reduce_rejects_mis_shaped_operands(no_launch):
    gen = torch.Generator(device="cuda").manual_seed(8)
    a = _attn(3, 4, 33, 36, gen)
    for g in (_attn(2, 4, 33, 36, gen), _attn(3, 3, 33, 36, gen), torch.randn(3, 4, 32, 32, device="cuda")):
        with pytest.raises(ValueError):
            ops.head_reduce(a, g, mode="mean")
    for w in (torch.randn(4, device="cuda"), torch.randn(2, 4, device="cuda"), torch.randn(3, 5, device="cuda"),
              torch.randn(12, device="cuda"), torch.randn(3, 4, 1, device="cuda")):
        with pytest.raises(ValueError):
            ops.head_reduce(a, head_weight=w, mode="mean_relu")


def test_heatmap_rejects_mis_shaped_maps(no_launch):
    for maps, grid in ((torch.randn(196, device="cuda"), 14), (torch.randn(2, 576, device="cuda"), 14),
                       (torch.randn(2, 195, device="cuda"), 14), (torch.randn(2, 14, 14, device="cuda"), 14),
                       (torch.randn(3, 196, device="cuda"), 24)):
        with pytest.raises(ValueError):
            visualization.relevance_to_heatmap(maps, grid=grid)
