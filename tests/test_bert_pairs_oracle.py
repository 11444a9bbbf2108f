"""CPU checks of sentence-pair BERT inputs (``token_type_ids``): the fp64 oracle with token types (``oracle/bert_pairs.py``)
reproduces the unmodified reference's fixture ``tests/golden/bert_pairs.npz`` (``oracle/make_golden_bert_pairs.py``), no
token types is exactly segment 0 and exactly ``oracle/bert.py``, and segment 1 changes the result, so the fixture
exercises the token-type table."""
import os

import numpy as np
import pytest
import torch

from oracle import attn_grad_rollout as agr
from oracle import bert as obert
from oracle import bert_pairs as opairs
from oracle import make_golden_bert_pairs as mgp


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "bert_pairs.npz"))


def _params(dt=torch.float64):
    params, heads = obert.init_params(**mgp.PARAMS)
    return {k: v.to(dt) for k, v in params.items()}, heads


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def test_fixture_inputs(golden):
    ids, mask, tt = mgp.pair_inputs()
    assert np.array_equal(golden["ids"], ids.numpy()) and np.array_equal(golden["mask"], mask.numpy())
    assert np.array_equal(golden["token_type_ids"], tt.numpy())
    assert int(golden["param_seed"]) == mgp.PARAM_SEED
    starts = [int(np.argmax(r == 1)) for r in golden["token_type_ids"]]
    assert len(set(starts)) == 3 and (golden["token_type_ids"][2] == 1).all(), "mixed boundaries, one all-segment-1 row"
    assert golden["mask"].min() == 0, "one row is padded"


def test_oracle_with_token_types_matches_reference_fixture(golden):
    p64, heads = _params()
    ids, mask, tt = mgp.pair_inputs()
    for s in range(ids.shape[0]):
        x, m, t = ids[s:s + 1], mask[s:s + 1], tt[s:s + 1]
        with torch.enable_grad():
            logits, cache = opairs.forward(p64, x, m, heads, need_grad=True, token_type_ids=t)
            seed = torch.zeros_like(logits)
            seed[0, logits.argmax(dim=-1)] = 1
            grads = obert.attention_gradients(cache, seed)
        key = "ours.f64.s%d" % s
        assert rel(logits.detach(), golden[key + ".logits"]) < 1e-12
        for lib in ("ours", "lrp"):
            assert np.array_equal(golden["%s.f64.s%d.logits" % (lib, s)], golden[key + ".logits"])
        for l in range(3):
            assert rel(cache["layers"][l]["probs"].detach(), golden["%s.attn.%d" % (key, l)]) < 1e-12
            assert rel(grads[l].detach(), golden["%s.grad.%d" % (key, l)]) < 1e-10
        for sl in (0, 1):
            out = opairs.explain(p64, x, m, heads, start_layer=sl, token_type_ids=t)[0]
            assert rel(out, golden["%s.LRP.sl%d" % (key, sl)]) < 1e-8
            assert torch.equal(out, torch.from_numpy(golden["oracle.s%d.LRP.sl%d" % (s, sl)]))
            agr_map = agr.bert_map([c["probs"].detach() for c in cache["layers"]], [g.detach() for g in grads], sl)
            assert torch.equal(agr_map, torch.from_numpy(golden["oracle.s%d.attn_grad_rollout.sl%d" % (s, sl)]))
            rollout, _ = opairs.explain_attn_grad_rollout(p64, x, m, heads, start_layer=sl, token_type_ids=t)
            assert torch.equal(rollout, agr_map)
        for which in obert.GENERATORS:
            for vt, kw in mgp.variants(which):
                ref = torch.from_numpy(golden["%s.%s.%s" % (key, which, vt)])
                out = opairs.generate(p64, x, m, heads, which, token_type_ids=t, **kw)
                assert torch.equal(torch.isnan(out), torch.isnan(ref)), (s, which, vt)
                if not torch.isnan(ref).any():
                    assert rel(out, ref) < 1e-8, (s, which, vt, rel(out, ref))
                assert torch.equal(torch.nan_to_num(out), torch.nan_to_num(
                    torch.from_numpy(golden["oracle.s%d.%s.%s" % (s, which, vt)])))


def test_fp32_reference_agrees_with_fp64(golden):
    """The fp32 fixture entries the GPU tests read are the reference's own fp32 results, close to its fp64 results."""
    for lib in ("ours", "lrp"):
        for s in range(3):
            key = "%s.%%s.s%d" % (lib, s)
            assert rel(golden[key % "f32" + ".logits"], golden[key % "f64" + ".logits"]) < 1e-5
            for sl in (0, 1):
                assert rel(golden[key % "f32" + ".LRP.sl%d" % sl], golden[key % "f64" + ".LRP.sl%d" % sl]) < 2e-2


@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_no_token_types_is_segment_zero_exactly(dt):
    params, heads = _params(dt)
    ids, mask, _ = mgp.pair_inputs()
    zeros = torch.zeros_like(ids)
    a, _ = opairs.forward(params, ids, mask, heads)
    b, _ = opairs.forward(params, ids, mask, heads, token_type_ids=zeros)
    assert torch.equal(a, b) and torch.equal(a, obert.forward(params, ids, mask, heads)[0])
    ma, ia = opairs.explain(params, ids, mask, heads, start_layer=0)
    mb, ib = opairs.explain(params, ids, mask, heads, start_layer=0, token_type_ids=zeros)
    m0, i0 = obert.explain(params, ids, mask, heads, start_layer=0)
    assert torch.equal(ma, mb) and torch.equal(ia, ib) and torch.equal(ma, m0) and torch.equal(ia, i0)
    for which in obert.GENERATORS:
        want = torch.nan_to_num(obert.generate(params, ids, mask, heads, which))
        assert torch.equal(torch.nan_to_num(opairs.generate(params, ids, mask, heads, which)), want)
        assert torch.equal(torch.nan_to_num(opairs.generate(params, ids, mask, heads, which, token_type_ids=zeros)), want)
    ra, _ = opairs.explain_attn_grad_rollout(params, ids, mask, heads, token_type_ids=zeros)
    assert torch.equal(ra, agr.explain_bert(params, ids, mask, heads)[0])
    assert obert.forward.__module__ == "oracle.bert", "segments() restores oracle.bert"


def test_segment_one_changes_the_result(golden):
    p64, heads = _params()
    ids, mask, tt = mgp.pair_inputs()
    a, _ = opairs.forward(p64, ids, mask, heads)
    b, _ = opairs.forward(p64, ids, mask, heads, token_type_ids=tt)
    assert (a - b).abs().min() > 1e-6, "every row has segment-1 tokens, so every row's logits move"
    assert rel(b[2:3], golden["ours.f64.s2.logits"]) < 1e-12
    assert rel(a[2:3], golden["ours.f64.s2.logits"]) > 1e-6
    ma, _ = opairs.explain(p64, ids[2:3], mask[2:3], heads, start_layer=0)
    mb, _ = opairs.explain(p64, ids[2:3], mask[2:3], heads, start_layer=0, token_type_ids=tt[2:3])
    assert rel(ma, mb) > 1e-6
