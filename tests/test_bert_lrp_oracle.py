"""CPU checks of the ``layers_lrp`` BERT classifier (``BERT_cls_lrp.py``): the oracle of ``tests/bert_lrp_oracle.py`` is
bit-exact to the reference's fixture ``tests/golden/bert_cls_lrp.npz`` (and to the live reference when it is present), the
facade modules resolve under the reference's import paths, and the facade's ``state_dict`` keys are the reference's."""
import os

import numpy as np
import pytest
import torch

import bert_lrp_oracle as olrp
from oracle import bert as obert
from oracle import ref_harness as rh

DTYPES = [("f32", torch.float32), ("f64", torch.float64)]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "bert_cls_lrp.npz"))


def _params(dt):
    params, heads = obert.init_params(rand_affine=True, **olrp.TINY)
    return {k: v.to(dt) for k, v in params.items()}, heads


def test_fixture_inputs_are_those_of_bert_generators(golden, golden_dir):
    g = np.load(os.path.join(golden_dir, "bert_generators.npz"))
    ids, mask = olrp.tiny_inputs()
    for z in (g, golden):
        assert np.array_equal(z["ids"], ids.numpy()) and np.array_equal(z["mask"], mask.numpy())
    assert int(golden["param_seed"]) == int(g["param_seed"])


@pytest.mark.parametrize("tag,dt", DTYPES)
def test_oracle_matches_fixture_bit_exact(golden, tag, dt):
    params, heads = _params(dt)
    ids, mask = olrp.tiny_inputs()
    for s in range(2):
        x, m = ids[s:s + 1], mask[s:s + 1]
        for which in olrp.GENERATORS:
            for name, kw in (("argmax", {}), ("index0", dict(index=0)), ("index1", dict(index=1))):
                ref = torch.from_numpy(golden["%s.s%d.%s.%s" % (tag, s, which, name)])
                out = olrp.generate(params, x, m, heads, which, **kw)
                assert out.dtype == ref.dtype and torch.equal(out, ref), "%s s%d %s %s" % (tag, s, which, name)
        for sl in (0, 1):
            row, _, taps = olrp.explain(params, x, m, heads, start_layer=sl, return_taps=True)
            assert torch.equal(row, torch.from_numpy(golden["%s.s%d.LRP.sl%d" % (tag, s, sl)])), "%s s%d sl%d" % (tag, s, sl)
            if sl == 0:
                for l in range(olrp.TINY["depth"]):
                    assert torch.equal(taps["cams"][l], torch.from_numpy(golden["%s.s%d.cam.%d" % (tag, s, l)]))


def test_padded_tokens_get_zero(golden):
    """the fixture's padded sample: no relevance reaches the padded tokens (-10000 keys) in either map"""
    for tag, _ in DTYPES:
        for which in olrp.GENERATORS:
            assert np.all(golden["%s.s1.%s.argmax" % (tag, which)][0, 18:] == 0)


def test_rules_differ_from_layers_ours(golden):
    """the two classifiers give different LRP maps on the same weights (why the separate model exists)"""
    params, heads = _params(torch.float64)
    ids, mask = olrp.tiny_inputs()
    ours = obert.generate(params, ids[:1], mask[:1], heads, "full_lrp")
    lrp = olrp.generate(params, ids[:1], mask[:1], heads, "full_lrp")
    assert (ours - lrp).abs().max() > 1e-3 * lrp.abs().max()


def test_batched_oracle_equals_per_sample():
    params, heads = _params(torch.float64)
    ids, mask = olrp.tiny_inputs()
    for which in olrp.GENERATORS:
        out = olrp.generate(params, ids, mask, heads, which)
        for s in range(2):
            one = olrp.generate(params, ids[s:s + 1], mask[s:s + 1], heads, which)
            assert torch.allclose(out[s], one[0], rtol=1e-12, atol=1e-14 * one.abs().max().item())


@pytest.mark.skipif(not rh.available(), reason="reference checkout not present")
def test_oracle_matches_live_reference():
    params, heads = _params(torch.float32)
    ids, mask = olrp.tiny_inputs()
    model = olrp._build_ref_cls_lrp(params, torch.float32)
    for which in olrp.GENERATORS:
        ref = rh.bert_generate(model, ids[1:2], mask[1:2], which)
        assert torch.equal(olrp.generate(params, ids[1:2], mask[1:2], heads, which), ref), which
    ref = rh.bert_generate_lrp(model, ids[1:2], mask[1:2], start_layer=0)["map"]
    assert torch.equal(olrp.explain(params, ids[1:2], mask[1:2], heads, start_layer=0)[0], ref)


def test_install_aliases_resolves_the_layers_lrp_modules():
    import sys
    import transformer_explainability_b200 as te
    te.install_aliases()
    from BERT_explainability.modules.BERT.BERT_cls_lrp import BertForSequenceClassification
    from BERT_explainability.modules.BERT.BERT_orig_lrp import BertModel, compute_rollout_attention  # noqa: F401
    from BERT_explainability.modules.layers_lrp import Linear, Add, MatMul, Mul, Tanh, Clone       # noqa: F401
    from transformer_explainability_b200._lib import FLAG_RULES_LRP
    base = "transformer_explainability_b200.BERT_explainability.modules."
    assert sys.modules["BERT_explainability.modules.BERT.BERT_cls_lrp"].__name__ == base + "BERT.BERT_cls_lrp"
    assert sys.modules["BERT_explainability.modules.BERT.BERT_orig_lrp"].__name__ == base + "BERT.BERT_orig_lrp"
    assert sys.modules["BERT_explainability.modules.layers_lrp"].__name__ == base + "layers_lrp"
    assert Linear.__module__ == "transformer_explainability_b200.modules.layers_lrp"
    cfg = type("C", (), dict(vocab_size=100, max_position_embeddings=32, type_vocab_size=2, hidden_size=64,
                             num_hidden_layers=2, num_attention_heads=4, intermediate_size=128, num_labels=2,
                             layer_norm_eps=1e-12))()
    m = BertForSequenceClassification(cfg)
    assert m._rule_flags == FLAG_RULES_LRP and m.engine_flags == 0


@pytest.mark.skipif(not rh.available(), reason="reference checkout not present")
def test_facade_state_dict_keys_equal_the_reference():
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import BertForSequenceClassification
    params, _ = _params(torch.float32)
    ref = olrp._build_ref_cls_lrp(params, torch.float32)
    cfg = type("C", (), dict(type_vocab_size=2, num_labels=2, layer_norm_eps=1e-12, **olrp.TINY_CFG))()
    ours = BertForSequenceClassification(cfg)
    assert set(ours.state_dict()) == set(ref.state_dict())
    ours.load_state_dict(ref.state_dict())
