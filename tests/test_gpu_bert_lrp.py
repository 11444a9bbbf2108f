"""The ``layers_lrp`` BERT classifier (``BERT_cls_lrp``) on the engine, and the ``layers_lrp`` Linear rule on the tensor
cores (``TE_FLAG_RULES_LRP_TC``).

- Tiny fixture (``bert_cls_lrp.npz``, the unmodified reference): every stored map within the bounds ``test_gpu_bert.py``
  uses for ``bert_generators.npz``, class index bit-exact, padded tokens exactly 0.
- ``ops.linear_relprop(variant="lrp_tc")`` at tensor-core shapes against fp64, and its zero pattern against the SIMT rule.
- A conditioned 3-layer BERT of BERT-base width (S = 130, batch 3, one row padded from the middle) against the fp64 oracle
  under five flag sets, the batched call against the per-sample calls, and the top-layer first-token-rows shortcut
  (strided rows) against the all-rows form, bit for bit.
- ``ViT_orig_LRP`` at ViT-B width with the tensor-core rule.
- The new column-fastest problems at one m-tile more than ``gridDim.y`` holds.

Measured on an H100 80GB HBM3 (400 W power limit), relative to the fp64 maximum: the ops-level rule 4.6e-5 ... 9.9e-5;
BERT-base width 1.0e-5 on the SIMT sets (0, 51 with the SIMT rule) and 2.2e-4 on the tensor-core sets; ``ViT_orig_LRP``
with the tensor-core rule 1.8e-3 (``full``, pixel maps).
"""
import os

import numpy as np
import pytest
import torch

import bert_lrp_oracle as olrp
from oracle import bert as obert
from oracle import conditioned
from oracle import cpu as ocpu
from oracle import rules
from transformer_explainability_b200 import _lib, ops

pytestmark = pytest.mark.gpu

TC = _lib.FLAG_RULES_LRP_TC
FLAG_SETS = [0, _lib.FLAG_ALL_FAST, _lib.FLAG_BENCH_DEFAULT, _lib.FLAG_BENCH_DEFAULT | TC,
             _lib.FLAG_BENCH_DEFAULT | _lib.FLAG_ZPLUS_R_F16 | _lib.FLAG_BACKWARD_F16 | TC]
GATE = 1e-4


def tol(flags):
    return 5e-3 if flags & (_lib.FLAG_TENSOR_CORES | TC) else 2e-4


def rel(a, b):
    b = torch.as_tensor(b).double().cpu()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def make_model(params, heads, **cfg):
    from transformers import BertConfig
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import \
        BertForSequenceClassification
    m = BertForSequenceClassification(BertConfig(num_attention_heads=heads, num_labels=2, **cfg))
    res = m.load_state_dict({k: v.float() for k, v in params.items()}, strict=False)
    assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
    return m.cuda().eval()


# ---- tiny fixture ----------------------------------------------------------------------------------------------------
TINY_TOL = {"LRP_last_layer": 2e-2, "full_lrp": 2e-2, "LRP": 2e-2}


@pytest.mark.parametrize("flags", [0, _lib.FLAG_BENCH_DEFAULT | TC])
def test_tiny_vs_reference_fixture(golden_dir, flags):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    g = np.load(os.path.join(golden_dir, "bert_cls_lrp.npz"))
    params, heads = obert.init_params(rand_affine=True, **olrp.TINY)
    cfg = {k: v for k, v in olrp.TINY_CFG.items() if k != "num_attention_heads"}
    model = make_model(params, heads, **cfg)
    model.engine_flags = flags
    gen = Generator(model)
    ids, mask = torch.from_numpy(g["ids"]), torch.from_numpy(g["mask"])
    logits32 = obert.forward(params, ids, mask, heads)[0]
    for key in [k for k in g.files if k.startswith("f32.") and k.split(".")[2] in TINY_TOL]:
        _, s, which, tag = key.split(".")
        s = int(s[1:])
        if which == "LRP":
            kw = {"start_layer": int(tag[2:])}
        else:
            kw = {} if tag == "argmax" else {"index": int(tag[5:])}
        out = getattr(gen, "generate_" + which)(ids[s:s + 1].cuda(), mask[s:s + 1].cuda(), **kw)
        torch.cuda.synchronize()
        ref = torch.from_numpy(g[key.replace("f32.", "f64.")])
        assert out.shape == ref.shape == (1, 24), key
        assert not torch.isnan(out).any(), key
        assert rel(out, ref) < TINY_TOL[which], "%s rel=%g" % (key, rel(out, ref))
        if "index" not in kw:
            assert int(model.engine().tensor("logits").argmax(-1)[0]) == int(logits32[s].argmax()), key
        if s == 1:
            assert float(out[0, 18:].abs().max()) == 0.0, "%s: padded tokens must get exactly zero" % key
    gen.generate_LRP(ids[:1].cuda(), mask[:1].cuda(), start_layer=0)
    for l in range(olrp.TINY["depth"]):                     # the attn_cam taps of generate_LRP(start_layer=0)
        cam = model.bert.encoder.layer[l].attention.self.get_attn_cam()
        assert rel(cam, g["f64.s0.cam.%d" % l]) < 2e-2


# ---- the tensor-core rule at the ops level -------------------------------------------------------------------------------
def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g) * scale


@pytest.mark.parametrize("rows,inf,outf", [(300, 256, 384), (129, 768, 768), (1000, 768, 3072), (77, 3072, 768)])
def test_lrp_tc_rule_vs_fp64(rows, inf, outf):
    x = _rand(rows, inf, seed=rows)
    w = _rand(outf, inf, seed=inf, scale=inf ** -0.5)
    r = _rand(rows, outf, seed=outf).abs_()
    out = ops.linear_relprop(x, w, r, variant="lrp_tc")
    ref = rules.linear_relprop_lrp(x.double().cpu(), w.double().cpu(), r.double().cpu())
    e = rel(out, ref)
    print("lrp_tc %dx%dx%d: %.1e" % (rows, inf, outf, e))
    assert e < 5e-3


def test_lrp_tc_rule_keeps_exact_zeros():
    rows, inf, outf = 260, 256, 384
    x = _rand(rows, inf, seed=1)
    x[3] = x[3].abs() + 0.1                 # no negative input: x- W-^T == 0, that half contributes exactly 0
    x[4] = -(x[4].abs() + 0.1)              # no positive input
    x[5] = 0                                # all-zero row
    x[:, 17] = 0                            # a zero input column
    w = _rand(outf, inf, seed=2, scale=inf ** -0.5)
    w[:, 40] = 0                            # a zero weight column: input 40 gets no relevance
    w[7] = w[7].abs()                       # an output with positive weights only
    r = _rand(rows, outf, seed=3).abs_()
    r[6] = 0                                # no relevance in row 6
    tc = ops.linear_relprop(x, w, r, variant="lrp_tc")
    simt = ops.linear_relprop(x, w, r, variant="lrp")
    torch.cuda.synchronize()
    assert torch.equal(tc == 0, simt == 0)
    for row in (5, 6):
        assert float(tc[row].abs().max()) == 0.0
    assert float(tc[:, 17].abs().max()) == 0.0 and float(tc[:, 40].abs().max()) == 0.0
    ref = rules.linear_relprop_lrp(x.double().cpu(), w.double().cpu(), r.double().cpu())
    assert rel(tc, ref) < 5e-3
    # the sign-free rows: only one half is non-zero, each within the TF32 bound of its fp64 value
    for row in (3, 4):
        assert rel(tc[row], ref[row]) < 5e-3


def test_lrp_tc_small_shapes_run_the_simt_rule():
    x, w = _rand(10, 64, seed=4), _rand(48, 64, seed=5, scale=0.125)
    r = _rand(10, 48, seed=6).abs_()
    assert torch.equal(ops.linear_relprop(x, w, r, variant="lrp_tc"), ops.linear_relprop(x, w, r, variant="lrp"))


# ---- conditioned BERT of BERT-base width ---------------------------------------------------------------------------------
CASES = [("LRP_last_layer", {}), ("full_lrp", {}), ("LRP", dict(start_layer=0)), ("LRP", dict(start_layer=1))]


def _cid(which, kw):
    return which + "".join(".%s=%s" % kv for kv in sorted(kw.items()))


@pytest.fixture(scope="module")
def bert_b():
    params, heads = obert.init_params(seed=22, vocab=1000, max_pos=512, dim=768, depth=3, heads=12, inter=3072,
                                      rand_affine=True)
    params = conditioned.condition_bert(params)
    g = torch.Generator().manual_seed(23)
    n, seq = 3, 130
    ids = torch.randint(5, 1000, (n, seq), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    mask = torch.ones(n, seq, dtype=torch.long)
    pad = seq // 2
    mask[1, pad:] = 0                                              # sample 1 is padded from the middle on
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    refs = {}
    for which, kw in CASES:
        if which == "LRP":
            ref, idx = olrp.explain(p64, ids, mask, heads, **kw)
            ref32, _ = olrp.explain(params, ids, mask, heads, **kw)
        else:
            ref, ref32, idx = (olrp.generate(p64, ids, mask, heads, which, **kw),
                               olrp.generate(params, ids, mask, heads, which, **kw), None)
        refs[_cid(which, kw)] = (ref, idx, rel(ref32, ref))
    ref = olrp.model_relprop(p64, ids, mask, heads)                    # model.relprop: relevance at the encoder input
    refs["relprop"] = (ref, None, rel(olrp.model_relprop(params, ids, mask, heads), ref))
    return dict(params=params, heads=heads, ids=ids, mask=mask, pad=pad, refs=refs,
                cfg=dict(hidden_size=768, num_hidden_layers=3, intermediate_size=3072, vocab_size=1000,
                         max_position_embeddings=512))


def test_bert_cls_lrp_every_case_every_flag_set(bert_b):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    for key, (_, _, e) in bert_b["refs"].items():
        assert e < GATE, "regime is not conditioned for %s: fp32 oracle vs fp64 oracle %g" % (key, e)
    model = make_model(bert_b["params"], bert_b["heads"], **bert_b["cfg"])
    gen = Generator(model)
    ids, mask, pad = bert_b["ids"].cuda(), bert_b["mask"].cuda(), bert_b["pad"]
    worst = {}
    for flags in FLAG_SETS:
        model.engine_flags = flags
        for which, kw in CASES:
            ref, ridx, _ = bert_b["refs"][_cid(which, kw)]
            out = getattr(gen, "generate_" + which)(ids, mask, **kw)
            torch.cuda.synchronize()
            assert out.shape == ref.shape and not torch.isnan(out).any()
            if ridx is not None:
                assert torch.equal(model.engine().tensor("logits").argmax(-1).cpu(), ridx), "%s: class index" % which
            assert float(out[1, pad:].abs().max()) == 0.0, "%s: padded tokens must get exactly zero" % which
            e = rel(out, ref)
            print("bert-cls-lrp %s flags %d: %.1e (bound %.0e)" % (_cid(which, kw), flags, e, tol(flags)))
            worst[tol(flags)] = max(worst.get(tol(flags), 0.0), e)
            assert e < tol(flags), "%s flags %d: %g" % (_cid(which, kw), flags, e)
        logits = model(ids, mask)[0]
        oh = torch.zeros_like(logits)
        oh[torch.arange(logits.shape[0]), logits.argmax(-1)] = 1
        r_in = model.relprop(oh, alpha=1)
        torch.cuda.synchronize()
        assert float(r_in[1, pad:].abs().max()) == 0.0
        e = rel(r_in, bert_b["refs"]["relprop"][0])
        print("bert-cls-lrp relprop flags %d: %.1e" % (flags, e))
        worst[tol(flags)] = max(worst.get(tol(flags), 0.0), e)
        assert e < tol(flags)
    print("worst", worst)
    # a batch is a set of independent sequences
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT | TC
    for which, kw in CASES:
        out = getattr(gen, "generate_" + which)(ids, mask, **kw)
        scale = out.abs().max().item()
        for s in range(ids.shape[0]):
            one = getattr(gen, "generate_" + which)(ids[s:s + 1], mask[s:s + 1], **kw)
            assert torch.allclose(one[0], out[s], rtol=1e-5, atol=1e-6 * scale), "%s: batched != per-sample" % which


def test_top_layer_first_token_rows_are_exact(bert_b):
    """the top layer's three Linear rules on the B first-token rows (strided x, r, out) equal the all-rows form bit for bit"""
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    model = make_model(bert_b["params"], bert_b["heads"], **bert_b["cfg"])
    gen = Generator(model)
    ids, mask = bert_b["ids"].cuda(), bert_b["mask"].cuda()
    lib = _lib.load()
    try:
        for flags in (0, _lib.FLAG_BENCH_DEFAULT | TC):
            model.engine_flags = flags
            outs = []
            for on in (1, 0):
                assert lib.te_set_option(b"cls_row_top_block", on) == 0
                outs.append(gen.generate_full_lrp(ids, mask).clone())
            assert torch.equal(outs[0], outs[1]), "flags %d" % flags
    finally:
        lib.te_set_option(b"cls_row_top_block", 1)


# ---- ViT_orig_LRP at ViT-B width -------------------------------------------------------------------------------------------
def test_vit_orig_lrp_tensor_core_rule():
    from test_gpu_methods_tc import ORIG_CASES, _run_vit_methods, _vit_model, _vit_setup
    setup = _vit_setup("vit_base_patch16_224", seed=15, xseed=16, cases=ORIG_CASES, variant="lrp")
    model = _vit_model(setup, module="ViT_orig_LRP")
    _run_vit_methods("vit-orig-lrp-tc", setup, model, [_lib.FLAG_ALL_FAST | TC, _lib.FLAG_BENCH_DEFAULT | TC])


# ---- column-fastest problems beyond gridDim.y ------------------------------------------------------------------------------
def test_lrp_tc_rule_tile_order():
    from test_gpu_tile_order import TALL, check_rows, rand
    x = rand(TALL, 128, seed=10)
    w = rand(128, 128, seed=11, scale=0.09)
    r = rand(TALL, 128, seed=12).abs_()
    check_rows(lambda xx, rr: ops.linear_relprop(xx, w, rr, variant="lrp_tc"), x, r)   # LrpSProb<+-> + LrpRProb<+->
