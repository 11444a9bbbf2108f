"""GPU: the LRP-alpha-beta rule (``relprop(R, alpha)``, beta = alpha - 1) on every Linear-rule path and through the engines.

- Rule level, alpha in {2, 0.5, 0}, against the fp64 oracle: every element's error over its own scale
  alpha |act| + |beta| |inh| (act, inh: the two halves in fp64; alpha * act - beta * inh can cancel, so |R_in| is no
  scale).  SIMT shapes (in / out not multiples of 128) 1e-5; at the ViT-B qkv / proj / fc1 / fc2 shapes the two-pass and
  single-pass TF32 paths, the S1-bf16 (2048) and fp16-R (8192) variants 3e-3, the bf16-R variant (64) 1.5e-2 (the bounds of
  tests/test_gpu_tc.py), the layers_lrp rule on SIMT 1e-5 and on TF32 tensor cores 3e-3.
- Conservation per row: sum R_in = sum R for layers_ours at every alpha (alpha - beta = 1); the layers_lrp row sums equal
  its alpha = 1 row sums.
- Engines at alpha = 2 against the fp64 oracle on the conditioned 3-block models of tests/test_gpu_methods_tc.py (its
  builders, FLAG_SETS, tol() and regime gate): every ViT method that reads the relprop, DeiT-distilled, ViT_orig_LRP
  (layers_lrp on SIMT and on tensor cores), BERT and BERT_cls_lrp relevance_in and attn_cam taps.
- The facades: Linear.relprop(R, alpha) of both libraries is ops.linear_relprop(alpha=...), model.relprop(alpha=2) is the
  engine's attribute(alpha=2), the alpha-independent rules ignore alpha, a NaN alpha raises.
"""
import pytest
import torch

import test_gpu_methods_tc as mtc
from oracle import alphabeta as ab
from oracle import bert as obert
from oracle import conditioned
from oracle import cpu as ocpu
from oracle import rules
from oracle import vit as ovit
from transformer_explainability_b200 import _lib, ops

pytestmark = pytest.mark.gpu

ALPHAS = (2.0, 0.5, 0.0)
VIT_SHAPES = [(394, 768, 2304), (394, 768, 768), (394, 768, 3072), (394, 3072, 768)]     # qkv, proj, fc1, fc2
SIMT_SHAPES = [(77, 200, 300), (130, 96, 250)]


def _inputs(rows, inf, outf, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, inf, generator=g)
    w = torch.randn(outf, inf, generator=g) * 0.05
    b = torch.randn(outf, generator=g)
    r = torch.rand(rows, outf, generator=g)
    return x, w, b, r


def _halves(x, w, r, lrp):
    """fp64 activator and inhibitor halves of the rule (R_in = alpha * act - beta * inh)"""
    x, w, r = x.double(), w.double(), r.double()
    px, nx, pw, nw = x.clamp(min=0), x.clamp(max=0), w.clamp(min=0), w.clamp(max=0)

    def f(w1, w2):
        if lrp:
            return px * (rules.safe_divide(r, px @ w1.t()) @ w1) + nx * (rules.safe_divide(r, nx @ w2.t()) @ w2)
        s = rules.safe_divide(r, px @ w1.t() + nx @ w2.t())
        return px * (s @ w1) + nx * (s @ w2)
    return f(pw, nw), f(nw, pw)


def _elem_err(out, x, w, r, alpha, lrp):
    act, inh = _halves(x, w, r, lrp)
    beta = alpha - 1
    ref = alpha * act - beta * inh
    scale = (alpha * act.abs() + abs(beta) * inh.abs()).clamp_min(1e-30)
    return ((out.double().cpu() - ref).abs() / scale).max().item(), ref


# (name, ops.linear_relprop kwargs, uses y / bias, lrp rule, bound)
TC_PATHS = [("tf32_two_pass", dict(tensor_cores=True), False, False, 3e-3),
            ("tf32_single_pass", dict(tensor_cores=True), True, False, 3e-3),
            ("bf16_r", dict(tensor_cores=True, bf16=True), True, False, 1.5e-2),
            ("bf16_s1", dict(tensor_cores=True, bf16="s1"), True, False, 3e-3),
            ("f16_r", dict(tensor_cores=True, bf16="s1", r_f16=True), True, False, 3e-3),
            ("lrp", dict(variant="lrp"), False, True, 1e-5),
            ("lrp_tc", dict(variant="lrp_tc"), False, True, 3e-3)]
SIMT_PATHS = [("simt", dict(), False, False, 1e-5), ("simt_y", dict(), True, False, 1e-5), ("lrp", dict(variant="lrp"), False, True, 1e-5)]


def _run_rule(rows, inf, outf, paths):
    x, w, b, r = _inputs(rows, inf, outf, rows + inf + outf)
    xd, wd, bd, rd = x.cuda(), w.cuda(), b.cuda(), r.cuda()
    y = ops.linear_forward(xd, wd, bd)
    for name, kw, with_y, lrp, bound in paths:
        extra = dict(y=y, bias=bd) if with_y else {}
        base = ops.linear_relprop(xd, wd, rd, **kw, **extra).double().cpu().sum(dim=1)
        for a in ALPHAS:
            out = ops.linear_relprop(xd, wd, rd, alpha=a, **kw, **extra)
            torch.cuda.synchronize()
            assert torch.isfinite(out).all()
            e, _ = _elem_err(out, x, w, r, a, lrp)
            print("%s rows %d in %d out %d alpha %g: %.2e per element (bound %.0e)" % (name, rows, inf, outf, a, e, bound))
            assert e < bound, (name, a, e)
            # conservation per row, within the rule's error over the per-row scale of the two halves
            sums = out.double().cpu().sum(dim=1)
            want = base if lrp else r.double().sum(dim=1)
            slack = bound * (a + abs(a - 1)) * (2 if lrp else 1) * r.double().sum(dim=1)
            assert ((sums - want).abs() <= slack).all(), (name, a, (sums - want).abs().max().item())


@pytest.mark.parametrize("rows,inf,outf", SIMT_SHAPES)
def test_rule_simt_shapes(rows, inf, outf):
    _run_rule(rows, inf, outf, SIMT_PATHS)


@pytest.mark.parametrize("rows,inf,outf", VIT_SHAPES)
def test_rule_vit_b_shapes(rows, inf, outf):
    _run_rule(rows, inf, outf, TC_PATHS)


def test_non_finite_alpha_raises():
    """a non-finite alpha is an argument error on every path"""
    x, w, b, r = _inputs(256, 768, 768, 5)
    xd, wd, rd = x.cuda(), w.cuda(), r.cuda()
    for kw in (dict(tensor_cores=True), dict(variant="lrp_tc"), dict()):
        for bad in (float("nan"), float("inf")):
            with pytest.raises(_lib.TeError):
                ops.linear_relprop(xd, wd, rd, alpha=bad, **kw)


# ---- engines at alpha = 2 against fp64 -----------------------------------------------------------------------------------
MODEL_ALPHA = 2.0
VIT_CASES = [c for c in mtc.VIT_CASES if c[0] != "last_layer_attn"]


def _vit_setup(name, seed, xseed, cases, variant="ours"):
    params, heads = ovit.init_params(name, seed=seed, rand_affine=True, depth=3, classes=100)
    params = conditioned.condition_vit(params, c_qkv=mtc.VIT_C_QKV)
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(xseed))
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    refs = {}
    for method, kw in cases:
        ref, idx = ab.vit_explain_method(p64, x.double(), heads, method, MODEL_ALPHA, variant=variant, **kw)
        ref32, _ = ab.vit_explain_method(params, x, heads, method, MODEL_ALPHA, variant=variant, **kw)
        refs[mtc._case_id(method, kw)] = (ref, idx, mtc.rel(ref32, ref))
    return dict(params=params, heads=heads, x=x, refs=refs, cases=cases)


@pytest.fixture(scope="module")
def vit_b():
    return _vit_setup("vit_base_patch16_224", seed=11, xseed=12, cases=VIT_CASES)


def _run_vit(tag, setup, model, flag_sets):
    x = setup["x"].cuda()
    for method, kw in setup["cases"]:
        e = setup["refs"][mtc._case_id(method, kw)][2]
        assert e < mtc.GATE, "regime is not conditioned for %s %s at alpha 2: fp32 oracle vs fp64 oracle %g" % (tag, method, e)
    for flags in flag_sets:
        model.engine_flags = flags
        for method, kw in setup["cases"]:
            ref, ridx, _ = setup["refs"][mtc._case_id(method, kw)]
            logits = model(x)
            oh = torch.zeros_like(logits)
            oh[torch.arange(logits.shape[0]), logits.argmax(-1)] = 1
            out = model.relprop(oh, method=method, alpha=MODEL_ALPHA, **kw)
            torch.cuda.synchronize()
            assert out.shape == ref.shape
            assert torch.equal(logits.argmax(-1).cpu(), ridx)
            mtc.record(tag, mtc._case_id(method, kw) + ".alpha2", flags, mtc.rel(out, ref), mtc.tol(flags))


def test_vit_methods_alpha2(vit_b):
    _run_vit("vit-b3", vit_b, mtc._vit_model(vit_b), mtc.FLAG_SETS)


def test_deit_alpha2():
    setup = _vit_setup("deit_base_distilled_patch16_224", seed=13, xseed=14, cases=mtc.DEIT_CASES)
    _run_vit("deit-b3", setup, mtc._vit_model(setup, distilled=True), mtc.FLAG_SETS)


def test_vit_orig_lrp_alpha2():
    setup = _vit_setup("vit_base_patch16_224", seed=15, xseed=16, cases=mtc.ORIG_CASES, variant="lrp")
    model = mtc._vit_model(setup, module="ViT_orig_LRP")
    _run_vit("vit-orig-lrp", setup, model, [0, _lib.FLAG_ALL_FAST | _lib.FLAG_RULES_LRP_TC])


def _bert_setup(seed, variant):
    params, heads = obert.init_params(seed=seed, vocab=1000, max_pos=512, dim=768, depth=3, heads=12, inter=3072,
                                      rand_affine=True)
    params = conditioned.condition_bert(params, c_qkv=3.0)
    g = torch.Generator().manual_seed(seed + 1)
    ids = torch.randint(5, 1000, (3, 130), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    mask = torch.ones(3, 130, dtype=torch.long)
    pad = 65
    mask[1, pad:] = 0
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    cams, r = ab.bert_model_relprop(p64, ids, mask, heads, MODEL_ALPHA, variant=variant)
    cams32, r32 = ab.bert_model_relprop(params, ids, mask, heads, MODEL_ALPHA, variant=variant)
    return dict(params=params, heads=heads, ids=ids, mask=mask, pad=pad, variant=variant, refs=(cams, r),
                gate=max([mtc.rel(r32, r)] + [mtc.rel(a, b) for a, b in zip(cams32, cams)]))


@pytest.fixture(scope="module")
def bert_b():
    return _bert_setup(22, "ours")


def _bert_model(setup, variant):
    cfg = dict(hidden_size=768, num_hidden_layers=3, intermediate_size=3072, vocab_size=1000, max_position_embeddings=512)
    if variant == "ours":
        from test_gpu_bert import make_model
    else:
        from test_gpu_bert_lrp import make_model
    return make_model(setup["params"], setup["heads"], **cfg)


def _run_bert(tag, setup, flag_sets):
    assert setup["gate"] < mtc.GATE, "regime is not conditioned for %s at alpha 2: %g" % (tag, setup["gate"])
    model = _bert_model(setup, setup["variant"])
    ids, mask = setup["ids"].cuda(), setup["mask"].cuda()
    cams, ref = setup["refs"]
    for flags in flag_sets:
        model.engine_flags = flags
        logits = model(ids, mask)[0]
        oh = torch.zeros_like(logits)
        oh[torch.arange(logits.shape[0]), logits.argmax(-1)] = 1
        r_in = model.relprop(oh, alpha=MODEL_ALPHA)
        torch.cuda.synchronize()
        assert r_in.shape == ref.shape and float(r_in[1, setup["pad"]:].abs().max()) == 0.0
        mtc.record(tag, "relevance_in.alpha2", flags, mtc.rel(r_in, ref), mtc.tol(flags))
        for l, layer in enumerate(model.bert.encoder.layer):
            mtc.record(tag, "attn_cam.%d.alpha2" % l, flags, mtc.rel(layer.attention.self.get_attn_cam(), cams[l]),
                       mtc.tol(flags))


def test_bert_alpha2(bert_b):
    _run_bert("bert-b3", bert_b, mtc.FLAG_SETS)


def test_bert_cls_lrp_alpha2():
    _run_bert("bert-cls-lrp", _bert_setup(23, "lrp"), [0, _lib.FLAG_ALL_FAST | _lib.FLAG_RULES_LRP_TC])


# ---- facades ---------------------------------------------------------------------------------------------------------------
def test_facades():
    from transformer_explainability_b200.modules import layers_lrp, layers_ours
    x, w, b, r = (t.cuda() for t in _inputs(64, 256, 384, 3))
    for mod, variant in ((layers_ours, "ours"), (layers_lrp, "lrp")):
        lin = mod.Linear(256, 384).cuda()
        with torch.no_grad():
            lin.weight.copy_(w)
            lin.bias.copy_(b)
        lin(x)
        assert torch.equal(lin.relprop(r, alpha=2), ops.linear_relprop(x, w, r, variant=variant, alpha=2.0))
        assert not torch.equal(lin.relprop(r, alpha=2), lin.relprop(r, alpha=1))
    # the rules that do not read alpha
    a1, a2 = torch.randn(2, 9, 32).cuda(), torch.randn(2, 9, 32).cuda()
    add = layers_ours.Add()
    add([a1, a2])
    ra = torch.randn(2, 9, 32).cuda()
    assert all(torch.equal(u, v) for u, v in zip(add.relprop(ra, alpha=2), add.relprop(ra, alpha=1)))
    cl = layers_ours.Clone()
    cl(a1, 2)
    assert torch.equal(cl.relprop((ra, a2), alpha=2), cl.relprop((ra, a2), alpha=1))
    e2 = layers_ours.einsum('bhij,bhjd->bhid')
    p, v = torch.rand(1, 2, 9, 9).softmax(-1).cuda(), torch.randn(1, 2, 9, 8).cuda()
    e2([p, v])
    rr = torch.randn(1, 2, 9, 8).cuda()
    assert all(torch.equal(u, q) for u, q in zip(e2.relprop(rr, alpha=2), e2.relprop(rr, alpha=1)))
    isel = layers_ours.IndexSelect()
    isel(a1, 1, torch.tensor(0).cuda())
    r1 = torch.randn(2, 1, 32).cuda()
    assert torch.equal(isel.relprop(r1, alpha=2), isel.relprop(r1, alpha=1))
    with pytest.raises(_lib.TeError):
        lin.relprop(r, alpha=float("nan"))


def test_model_relprop_equals_engine_attribute(vit_b):
    model = mtc._vit_model(vit_b)
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT
    x = vit_b["x"].cuda()
    logits = model(x)
    oh = torch.zeros_like(logits)
    oh[torch.arange(2), logits.argmax(-1)] = 1
    out = model.relprop(oh, alpha=2).clone()
    maps, _ = model.engine().attribute(index=logits.argmax(-1).to(torch.int32), alpha=2.0)
    assert torch.equal(out, maps)
    with pytest.raises(_lib.TeError):
        model.relprop(oh, alpha=float("nan"))
