"""CPU: the LRP-alpha-beta rule (``relprop(R, alpha)``, alpha != 1) of the oracle against the unmodified reference's
outputs in ``tests/golden/alphabeta.npz`` (``oracle/make_golden_alphabeta.py``), bit-exact in fp32 and fp64: the Linear
rule of both rule libraries and their BERT copies, ``model.relprop(alpha=2)`` of ViT / ViT_orig_LRP for every method that
reads the relprop, and of the BERT classifiers of both libraries.  At alpha = 1 the oracle is the z+ rule it always was."""
import os

import numpy as np
import pytest
import torch

from oracle import alphabeta as ab
from oracle import bert as obert
from oracle import rules
from oracle.make_golden_alphabeta import ALPHAS, MODEL_ALPHA, ORIG_METHODS, VIT_METHODS, _bert_cases, rule_inputs

DTYPES = [("f32", torch.float32), ("f64", torch.float64)]


def T(a):
    return torch.from_numpy(np.asarray(a))


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "alphabeta.npz"))


def test_fixture_inputs_are_regenerated_from_seeds(golden):
    x, w, r = rule_inputs()
    assert torch.equal(x, T(golden["rule.x"])) and torch.equal(w, T(golden["rule.w"])) and torch.equal(r, T(golden["rule.r"]))
    assert tuple(golden["alphas"]) == ALPHAS and float(golden["model_alpha"]) == MODEL_ALPHA
    ids, mask, _ = _bert_cases()
    assert np.array_equal(golden["bert.ids"], ids.numpy()) and np.array_equal(golden["bert.mask"], mask.numpy())


@pytest.mark.parametrize("tag,dt", DTYPES)
def test_linear_rules_match_reference(golden, tag, dt):
    x, w, r = (t.to(dt) for t in rule_inputs())
    for lib, fn in (("ours", ab.linear_relprop), ("lrp", ab.linear_relprop_lrp),
                    ("bert_ours", ab.linear_relprop), ("bert_lrp", ab.linear_relprop_lrp)):
        for a in ALPHAS:
            out = fn(x, w, r, alpha=a)
            assert out.dtype == dt and torch.equal(out, T(golden["%s.rule.%s.a%s" % (tag, lib, a)])), (lib, a)


@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_alpha_one_is_the_z_plus_rule(dt):
    """alpha = 1 (int or float) computes exactly what the oracle computed before alpha existed (the z+ closed forms)."""
    g = torch.Generator().manual_seed(3)
    x, w = torch.randn(6, 9, generator=g).to(dt), torch.randn(5, 9, generator=g).to(dt)
    r = torch.rand(6, 5, generator=g).to(dt)
    px, nx, pw, nw = x.clamp(min=0), x.clamp(max=0), w.clamp(min=0), w.clamp(max=0)
    s = rules.safe_divide(r, px @ pw.t() + nx @ nw.t())
    zplus = px * (s @ pw) + nx * (s @ nw)
    s1, s2 = rules.safe_divide(r, px @ pw.t()), rules.safe_divide(r, nx @ nw.t())
    lrp = px * (s1 @ pw) + nx * (s2 @ nw)
    for a in (1, 1.0):
        assert torch.equal(ab.linear_relprop(x, w, r, alpha=a), zplus)
        assert torch.equal(ab.linear_relprop_lrp(x, w, r, alpha=a), lrp)
    assert torch.equal(rules.linear_relprop(x, w, r), zplus) and torch.equal(rules.linear_relprop_lrp(x, w, r), lrp)
    with ab.alpha_rules(2):                               # the binding is undone on leaving the block
        pass
    assert torch.equal(rules.linear_relprop(x, w, r), zplus) and rules.add_relprop is not rules.add_relprop_simple


@pytest.mark.parametrize("dt", [torch.float64])
def test_conservation_at_any_alpha(dt):
    """alpha - beta = 1: each layers_ours row keeps its relevance at any alpha (no zero denominator here); the layers_lrp
    rule's row sums do not depend on alpha (each of its four products conserves its share of R on its own).  Up to the
    1e-9 that safe_divide adds to every denominator."""
    g = torch.Generator().manual_seed(5)
    x, w = torch.randn(4, 16, generator=g).to(dt), torch.randn(12, 16, generator=g).to(dt)
    r = torch.rand(4, 12, generator=g).to(dt)
    base = rules.linear_relprop_lrp(x, w, r).sum(dim=1)
    for a in ALPHAS:
        assert torch.allclose(ab.linear_relprop(x, w, r, alpha=a).sum(dim=1), r.sum(dim=1), rtol=1e-7, atol=0)
        assert torch.allclose(ab.linear_relprop_lrp(x, w, r, alpha=a).sum(dim=1), base, rtol=1e-7, atol=0)


@pytest.mark.parametrize("tag,dt", DTYPES)
def test_vit_model_relprop_matches_reference(golden, tag, dt):
    from oracle import vit as ovit
    params, heads = ovit.init_params("vit_tiny_test", seed=1, rand_affine=True)
    params = {k: v.to(dt) for k, v in params.items()}
    xs = T(golden["vit.x"]).to(dt)
    assert heads == int(golden["vit.heads"])
    n = 0
    for name, variant, methods in (("vit", "ours", VIT_METHODS), ("orig", "lrp", {m: (m, False) for m in ORIG_METHODS})):
        for s in range(xs.shape[0]):
            for key, (method, abl) in methods.items():
                out, _ = ab.vit_explain_method(params, xs[s:s + 1], heads, method, MODEL_ALPHA, is_ablation=abl,
                                               variant=variant)
                assert torch.equal(out, T(golden["%s.%s.s%d.%s" % (tag, name, s, key)]).reshape(out.shape)), (name, s, key)
                n += 1
            _, _, taps = ab.vit_explain(params, xs[s:s + 1], heads, MODEL_ALPHA, return_taps=True, variant=variant)
            for l in range(3):
                assert torch.equal(taps["cams"][l], T(golden["%s.%s.s%d.cam.%d" % (tag, name, s, l)])), (name, s, l)
    assert n == 2 * (len(VIT_METHODS) + len(ORIG_METHODS))


@pytest.mark.parametrize("tag,dt", DTYPES)
def test_bert_model_relprop_matches_reference(golden, tag, dt):
    """BertForSequenceClassification (layers_ours) and BERT_cls_lrp (layers_lrp) model.relprop(alpha=2): relevance at the
    encoder input and attn_cam of every layer, one full and one padded sequence."""
    ids, mask, cases = _bert_cases()
    for name, params, _, _ in cases:
        p = {k: v.to(dt) for k, v in params.items()}
        for s in range(2):
            cams, r = ab.bert_model_relprop(p, ids[s:s + 1], mask[s:s + 1], 4, MODEL_ALPHA,
                                            variant="lrp" if name == "cls_lrp" else "ours")
            assert torch.equal(r, T(golden["%s.%s.s%d.r" % (tag, name, s)])), (name, s)
            for l in range(3):
                assert torch.equal(cams[l], T(golden["%s.%s.s%d.cam.%d" % (tag, name, s, l)])), (name, s, l)


def test_bert_oracle_lrp_variant_is_the_cls_lrp_oracle():
    """at alpha = 1 the variant="lrp" relprop of oracle.alphabeta is what tests/bert_lrp_oracle.py restates, and the
    layers_ours one is oracle.bert's"""
    import bert_lrp_oracle as olrp
    params, heads = obert.init_params(rand_affine=True, **olrp.TINY)
    params = {k: v.double() for k, v in params.items()}
    ids, mask = olrp.tiny_inputs()
    want = olrp.model_relprop(params, ids, mask, heads)
    _, got = ab.bert_model_relprop(params, ids, mask, heads, 1, variant="lrp")
    assert torch.equal(got, want)
    _, got = ab.bert_model_relprop(params, ids, mask, heads, 1)
    with torch.no_grad():
        logits, cache = obert.forward(params, ids, mask, heads)
        seed = torch.nn.functional.one_hot(logits.argmax(-1), logits.shape[-1]).to(logits.dtype)
        _, want = obert.relprop(params, cache, seed, lowest=0, to_input=True)
    assert torch.equal(got, want)
