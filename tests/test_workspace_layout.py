"""CPU: every workspace region an engine lends to a kernel is at least as large as that kernel's use of it.

The ViT and BERT engines keep a few scratch regions (``tmp_f0/1`` [M, F], ``tmp_3d0/1`` [M, 3D], M = batch * tokens) and
lend them to kernels that run while they are idle: the hi-only fp16 split of the output gradient of every backward Linear
(``TE_FLAG_BACKWARD_F16``, rows * out / 2 floats, scales rows * ceil(out / 128) floats), the ``|x|`` scratch of the
single-pass z+ rules ([rows, in]), the 3-way clone's sum.  Those uses are not all F wide: the qkv backward splits a 3D-wide
gradient, the qkv z+ rule a D-wide input.  So with mlp_ratio < 1.5 a region sized M * F would be overrun, and the kernel
would write into the next region, which may be the very tensor it is reading.  The regions are laid out back to back,
so the extent of one is the distance to the next; ``te_*_tensor`` computes the views on the host without touching a
device, with any 256-byte-aligned address as the workspace.
"""
import ctypes

import pytest

from transformer_explainability_b200 import _lib
from transformer_explainability_b200.engine import bert_config, vit_config

FAKE_WS = 1 << 40                                    # 256-byte aligned; never dereferenced


def _views(lib, fn, cfg, *shape):
    out = {}
    for name in ("tmp_f0", "tmp_f1", "tmp_3d0", "tmp_3d1"):
        p, dims, strides = ctypes.c_void_p(), (ctypes.c_longlong * 4)(), (ctypes.c_longlong * 4)()
        assert fn(ctypes.byref(cfg), *shape, ctypes.c_void_p(FAKE_WS), name.encode(), 0, ctypes.byref(p), dims,
                  strides) == 0, lib.te_last_error()
        numel = 1
        for d in dims:
            numel *= d
        out[name] = (p.value, numel)
    return out


def _extents(views):
    """floats from each region to the next one in the carve order; the last is known only by its view"""
    order = ["tmp_f0", "tmp_f1", "tmp_3d0", "tmp_3d1"]
    ext = {}
    for a, b in zip(order, order[1:]):
        assert views[b][0] > views[a][0]
        ext[a] = (views[b][0] - views[a][0]) // 4
    ext["tmp_3d1"] = views["tmp_3d1"][1]
    return ext


def _bwd_split_uses(M, D, F):
    """(split floats, scale floats) of the hi-only fp16 split of dy of each backward Linear: fc2, fc1, proj, qkv"""
    return [(M * out // 2, M * -(-out // 128)) for out in (D, F, D, 3 * D)]


def _check(ext, uses):
    for region, need, what in uses:
        assert ext[region] >= need, "%s: %d floats, %s needs %d" % (region, ext[region], what, need)


VIT = [dict(embed_dim=256, num_heads=4, mlp_ratio=r) for r in (0.5, 1.0, 1.5, 2.0, 4.0)] + \
      [dict(embed_dim=256, num_heads=4, mlp_ratio=1.0, distilled=True), dict(), dict(embed_dim=768, mlp_ratio=1.0)] + \
      [dict(embed_dim=192, num_heads=3), dict(embed_dim=384, num_heads=6), dict(embed_dim=384, num_heads=6, distilled=True),
       dict(embed_dim=384, num_heads=12), dict(embed_dim=384, num_heads=8), dict(img_size=384)]     # tests/test_gpu_model_geometries.py


@pytest.mark.parametrize("kw", VIT, ids=lambda kw: "-".join("%s%s" % (k, v) for k, v in kw.items()) or "vit_b16")
@pytest.mark.parametrize("batch", [1, 3])
def test_vit_lent_regions_cover_their_uses(kw, batch):
    lib = _lib.load()
    cfg = vit_config(**kw)
    D, F = cfg.dim, cfg.mlp_dim
    npatch = (cfg.img_size // cfg.patch_size) ** 2
    M = batch * (npatch + (2 if cfg.distilled else 1))
    ext = _extents(_views(lib, lib.te_vit_tensor, cfg, batch))
    uses = [("tmp_f0", M * F, "dF / RF"),
            ("tmp_f0", batch * npatch * cfg.in_chans * cfg.patch_size ** 2, "the im2col patches"),
            ("tmp_f0", M * D, "the |x| scratch of the qkv z+ rule"),
            ("tmp_f1", M * F, "SF, the |x| scratch of the fc2 z+ rule, the GELU-output fp16 split"),
            ("tmp_3d0", M * 3 * D, "dqkv / S of the qkv z+ rule"),
            ("tmp_3d0", 2 * M * D, "the |x| scratch of the proj z+ rule at S + M*D")]
    for split, scale in _bwd_split_uses(M, D, F):
        uses += [("tmp_f1", split, "the fp16 split of dy"), ("tmp_3d1", scale, "the block scales of dy")]
    _check(ext, uses)


BERT = [dict(hidden_size=256, num_attention_heads=4, intermediate_size=f) for f in (128, 256, 384, 512, 1024)] + \
       [dict(), dict(intermediate_size=768)] + \
       [dict(hidden_size=128, num_attention_heads=2, intermediate_size=512),
        dict(hidden_size=384, num_attention_heads=12, intermediate_size=1536),
        dict(hidden_size=512, num_attention_heads=8, intermediate_size=2048)]         # tests/test_gpu_model_geometries.py


@pytest.mark.parametrize("kw", BERT, ids=lambda kw: "-".join("%s%s" % (k, v) for k, v in kw.items()) or "bert_base")
@pytest.mark.parametrize("batch,seq", [(1, 130), (3, 512)])
def test_bert_lent_regions_cover_their_uses(kw, batch, seq):
    lib = _lib.load()
    cfg = bert_config(**kw)
    D, F, M = cfg.hidden, cfg.intermediate, batch * seq
    ext = _extents(_views(lib, lib.te_bert_tensor, cfg, batch, seq))
    uses = [("tmp_f0", M * F, "dF / RF"),
            ("tmp_f1", M * F, "SF, the |x| scratch of the output-dense z+ rule, the GELU-output fp16 split"),
            ("tmp_f1", M * D, "the 3-way clone's sum"),
            ("tmp_3d0", M * 3 * D, "dqkv / S"),
            ("tmp_3d0", 2 * M * D, "the |x| scratch of the attention z+ rules at S + M*D")]
    for split, scale in _bwd_split_uses(M, D, F):
        uses += [("tmp_f1", split, "the fp16 split of dy"), ("tmp_3d1", scale, "the block scales of dy")]
    _check(ext, uses)


# ---- the saved-activation taps: documented views, inside the workspace, disjoint --------------------------------------------
SCRATCH = ["tmp_d%d" % i for i in range(4)] + ["tmp_f0", "tmp_f1", "tmp_3d0", "tmp_3d1"]


def _tap(fn, cfg, shape, name, layer):
    p, dims, strides = ctypes.c_void_p(), (ctypes.c_longlong * 4)(), (ctypes.c_longlong * 4)()
    rc = fn(ctypes.byref(cfg), *shape, ctypes.c_void_p(FAKE_WS), name.encode(), layer, ctypes.byref(p), dims, strides)
    assert rc == 0, name
    return p.value, tuple(dims), tuple(strides)


def _rows(B, N, W):
    """[B, N, W] row-major, padded to four dims"""
    return (B, N, W, 1), (N * W, W, 1, 1)


def _check_taps(fn, cfg, shape, nbytes, per_layer, per_model, depth):
    """every tap has its documented dims / strides, lies inside the workspace, and no two saved taps (nor a saved tap and
    the lent scratch) share a byte"""
    spans = []
    for layer, table in [(l, per_layer) for l in range(depth)] + [(0, per_model)]:
        for name, (dims, strides) in table.items():
            p, d, s = _tap(fn, cfg, shape, name, layer)
            assert (d, s) == (dims, strides), "%s[%d]: dims %s strides %s" % (name, layer, d, s)
            extent = 1 + sum((n - 1) * st for n, st in zip(d, s))
            assert FAKE_WS <= p and p + 4 * extent <= FAKE_WS + nbytes, "%s[%d] outside the workspace" % (name, layer)
            spans.append((p, p + 4 * extent, "%s[%d]" % (name, layer)))
    for name in SCRATCH:
        p, d, s = _tap(fn, cfg, shape, name, 0)
        spans.append((p, p + 4 * (1 + sum((n - 1) * st for n, st in zip(d, s))), name))
    spans.sort()
    for (a0, a1, an), (b0, b1, bn) in zip(spans, spans[1:]):
        assert a1 <= b0, "%s overlaps %s" % (an, bn)


@pytest.mark.parametrize("kw", VIT, ids=lambda kw: "-".join("%s%s" % (k, v) for k, v in kw.items()) or "vit_b16")
@pytest.mark.parametrize("batch", [1, 3])
def test_vit_taps_in_bounds_and_disjoint(kw, batch):
    lib = _lib.load()
    cfg = vit_config(**kw)
    B, D, F, H, C = batch, cfg.dim, cfg.mlp_dim, cfg.heads, cfg.num_classes
    N = (cfg.img_size // cfg.patch_size) ** 2 + (2 if cfg.distilled else 1)
    NP = (N + 3) & ~3
    att = ((B, H, N, N), (H * N * NP, N * NP, NP, 1))
    per_layer = dict(attn=att, attn_grad=att, attn_cam=att, qkv=_rows(B, N, 3 * D), h=_rows(B, N, F), g=_rows(B, N, F))
    per_layer.update({n: _rows(B, N, D) for n in ("x_in", "xn1", "ctx", "attn_out", "x_mid", "xn2", "mlp_out")})
    per_layer.update({n: ((B, N, 1, 1), (N, 1, 1, 1)) for n in ("mean1", "rstd1", "mean2", "rstd2")})
    per_model = dict(x_last=_rows(B, N, D), x_final_norm=_rows(B, N, D), logits=((B, C, 1, 1), (C, 1, 1, 1)),
                     rollout_mats=((cfg.depth, B, N, N), (B * N * NP, N * NP, NP, 1)))
    nbytes = lib.te_vit_workspace_bytes(ctypes.byref(cfg), batch)
    _check_taps(lib.te_vit_tensor, cfg, (batch,), nbytes, per_layer, per_model, cfg.depth)


@pytest.mark.parametrize("kw", BERT, ids=lambda kw: "-".join("%s%s" % (k, v) for k, v in kw.items()) or "bert_base")
@pytest.mark.parametrize("batch,seq", [(1, 130), (3, 512)])
def test_bert_taps_in_bounds_and_disjoint(kw, batch, seq):
    lib = _lib.load()
    cfg = bert_config(**kw)
    B, N, D, F, H, C = batch, seq, cfg.hidden, cfg.intermediate, cfg.heads, cfg.num_labels
    NP = (N + 3) & ~3
    att = ((B, H, N, N), (H * N * NP, N * NP, NP, 1))
    per_layer = dict(attn=att, attn_grad=att, attn_cam=att, qkv=_rows(B, N, 3 * D), hpre=_rows(B, N, F), g=_rows(B, N, F))
    per_layer.update({n: _rows(B, N, D) for n in ("hidden", "ctx", "d1", "s1", "ao", "d2", "s2")})
    per_layer.update({n: ((B, N, 1, 1), (N, 1, 1, 1)) for n in ("mean1", "rstd1", "mean2", "rstd2")})
    per_model = dict(h_last=_rows(B, N, D), pooled=((B, D, 1, 1), (D, 1, 1, 1)), logits=((B, C, 1, 1), (C, 1, 1, 1)))
    nbytes = lib.te_bert_workspace_bytes(ctypes.byref(cfg), batch, seq)
    _check_taps(lib.te_bert_tensor, cfg, (batch, seq), nbytes, per_layer, per_model, cfg.layers)


# te_*_workspace_bytes of the benchmarked configurations (batch 1 and the benchmarked batch), as laid out before the
# lent regions were sized by their uses: with F = 4D every use fits in M*F, so the size must not move
BASELINE_BYTES = [
    ("vit", dict(), 1, 218101760),
    ("vit", dict(), 256, 55828030464),
    ("vit", dict(embed_dim=1024, depth=24, num_heads=16), 1, 556246272),
    ("vit", dict(embed_dim=1024, depth=24, num_heads=16), 64, 35597718272),
    ("vit", dict(distilled=True), 1, 219188224),
    ("vit", dict(distilled=True), 256, 56107475968),
    ("bert", dict(), (1, 512), 862579712),
    ("bert", dict(), (64, 512), 55205061632),
]


@pytest.mark.parametrize("model,kw,shape,nbytes", BASELINE_BYTES)
def test_baseline_workspace_bytes_unchanged(model, kw, shape, nbytes):
    lib = _lib.load()
    if model == "vit":
        assert lib.te_vit_workspace_bytes(ctypes.byref(vit_config(**kw)), shape) == nbytes
    else:
        assert lib.te_bert_workspace_bytes(ctypes.byref(bert_config(**kw)), *shape) == nbytes
