"""GPU: the BERT engine (C ABI behind the reference-shaped Generator / BertForSequenceClassification facade) vs the
reference's stored outputs (tests/golden/bert_tiny.npz) and the fp64 oracle.

Maps are row 0 of a row-normalised rollout whose element 0 is replaced by the row minimum, so their maximum is
tiny (~1e-8 at random init); tolerances are relative to the map maximum."""
import os

import numpy as np
import pytest
import torch

from oracle import bert as obert
from oracle import cpu as ocpu

pytestmark = pytest.mark.gpu


def T(a):
    return torch.from_numpy(np.asarray(a))


def rel(a, b):
    b = torch.as_tensor(b).double()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def make_model(params, heads, **cfg):
    from transformers import BertConfig
    from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
        BertForSequenceClassification
    m = BertForSequenceClassification(BertConfig(num_attention_heads=heads, num_labels=2, **cfg))
    res = m.load_state_dict({k: v.float() for k, v in params.items()}, strict=False)
    assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
    return m.cuda().eval()


TINY = dict(hidden_size=64, num_hidden_layers=3, intermediate_size=128, vocab_size=100, max_position_embeddings=32)


def test_bert_tiny_vs_golden_reference(golden_dir):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    g = np.load(os.path.join(golden_dir, "bert_tiny.npz"))
    params = {k[len("param."):]: T(g[k]) for k in g.files if k.startswith("param.")}
    model = make_model(params, int(g["heads"]), **TINY)
    gen = Generator(model)
    ids, mask = T(g["ids"]).cuda(), T(g["mask"]).cuda()
    for s in range(2):
        for sl in (0, 1, 2):
            out = gen.generate_LRP(ids[s:s + 1], mask[s:s + 1], start_layer=sl)
            ref = T(g["f64.s%d.map.sl%d" % (s, sl)])
            assert out.shape == ref.shape == (1, 24)
            assert rel(out, ref) < 2e-2, "bert tiny s=%d sl=%d rel=%g" % (s, sl, rel(out, ref))
        out = gen.generate_LRP(ids[s:s + 1], mask[s:s + 1], start_layer=0)
        logits = model._engine.tensor("logits")
        assert rel(logits, T(g["f64.s%d.logits" % s])) < 1e-5
        assert int(logits.argmax()) == int(T(g["f64.s%d.logits" % s]).argmax())
        layers = model.bert.encoder.layer
        for l in range(3):
            assert rel(layers[l].attention.self.get_attn(), T(g["f64.s%d.attn.%d" % (s, l)])) < 1e-5
            assert rel(layers[l].attention.self.get_attn_gradients(), T(g["f64.s%d.grad.%d" % (s, l)])) < 1e-4
            assert rel(layers[l].attention.self.get_attn_cam(), T(g["f64.s%d.cam.%d" % (s, l)])) < 2e-2
    out = gen.generate_LRP(ids[0:1], mask[0:1], index=0, start_layer=0)
    assert rel(out, T(g["f64.s0.map.index0"])) < 2e-2
    # padded tokens get exactly zero relevance (mask = 0 from position 18 on in sample 1)
    out = gen.generate_LRP(ids[1:2], mask[1:2], start_layer=0)
    assert float(out[0, 18:].abs().max()) == 0.0
    # default start_layer=11 of the reference signature is out of range for a 3-layer model -> error, not garbage
    with pytest.raises(RuntimeError):
        gen.generate_LRP(ids[0:1], mask[0:1])


def test_bert_tiny_batched_and_relprop_api(golden_dir):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    params, heads = obert.init_params(seed=5, vocab=100, max_pos=32, dim=64, depth=3, heads=4, inter=128,
                                      rand_affine=True)
    model = make_model(params, heads, **TINY)
    gen = Generator(model)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(5, 100, (4, 20), generator=g)
    mask = torch.ones(4, 20, dtype=torch.long)
    mask[2, 15:] = 0
    maps, idx = gen.generate_LRP_batched(ids.cuda(), mask.cuda(), start_layer=0, return_index=True)
    ref, ridx = obert.explain({k: v.double() for k, v in params.items()}, ids, mask, heads, start_layer=0)
    assert torch.equal(idx.cpu().long(), ridx)
    for s in range(4):
        assert rel(maps[s], ref[s]) < 2e-2
        one = gen.generate_LRP(ids[s:s + 1].cuda(), mask[s:s + 1].cuda(), start_layer=0)
        assert torch.allclose(one[0], maps[s], rtol=1e-5, atol=1e-12)
    # model(...)[0] / model.relprop(one_hot, alpha=1): relevance at the encoder input is conserved (sums to 1)
    logits = model(ids[:1].cuda(), mask[:1].cuda())[0]
    oh = torch.zeros_like(logits)
    oh[0, logits.argmax()] = 1
    r_in = model.relprop(oh, alpha=1)
    assert r_in.shape == (1, 20, 64)
    assert abs(r_in.double().sum().item() - 1.0) < 1e-3


@pytest.mark.parametrize("seq,start", [(128, 0), (512, 11)])
def test_bert_base_vs_oracle(seq, start):
    """BERT-base (BASELINE configs[4] shape; S=512 with the pipeline default start_layer=11, S=128 with the notebook's
    start_layer=0), fp32 SIMT and tensor-core z+ paths.

    At random init the reference itself is badly conditioned on this model: its fp32 result (== oracle fp32, bit-equal)
    deviates from its fp64 result by 2e-2 ... 7e-1 of the map maximum depending on the thread count (measured,
    DESIGN.md §2).  So: class index bit-exact; logits, attention gradients and the top layer's attn_cam (one block of
    relprop, little amplification) tight; final maps judged against the reference's own fp32-vs-fp64 error
    measured on this box: median(err_new) <= max(5e-2, 3 * median(err_ref))."""
    from transformer_explainability_b200 import _lib
    params, heads = obert.init_params(seed=0, rand_affine=True)
    model = make_model(params, heads)
    eng = model.engine()
    g = torch.Generator().manual_seed(seq)
    n = 3
    ids = torch.randint(1000, 5000, (n, seq), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    mask = torch.ones(n, seq, dtype=torch.long)
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    ref, ridx, taps = obert.explain(p64, ids, mask, heads, start_layer=start, return_taps=True)
    ref32, _ = obert.explain(params, ids, mask, heads, start_layer=start)
    err_ref = sorted(rel(ref32[s], ref[s]) for s in range(n))
    top = len(taps["cams"]) - 1
    for flags in (0, _lib.FLAG_ZPLUS_TENSOR_CORES, _lib.FLAG_ALL_FAST):
        maps, idx, logits = eng.explain(ids.cuda(), mask.cuda(), start_layer=start, flags=flags, return_logits=True)
        assert torch.equal(idx.cpu().long(), ridx)
        assert rel(logits, taps["logits"]) < 1e-4
        layers = model.bert.encoder.layer
        assert rel(layers[top].attention.self.get_attn_gradients(), taps["grads"][top]) < 1e-3
        assert rel(layers[start].attention.self.get_attn_gradients(), taps["grads"][start]) < 1e-3
        cam_err = sorted(rel(layers[top].attention.self.get_attn_cam()[s], taps["cams"][top][s]) for s in range(n))
        errs = sorted(rel(maps[s], ref[s]) for s in range(n))
        print("bert-base S=%d start=%d flags=%d: top-cam rel %s | map rel %s | reference fp32-vs-fp64 %s" % (
            seq, start, flags, ["%.1e" % e for e in cam_err], ["%.1e" % e for e in errs], ["%.1e" % e for e in err_ref]))
        assert cam_err[n // 2] < 5e-2
        assert errs[n // 2] <= max(5e-2, 3 * err_ref[n // 2])


def test_bert_comparison_generators_vs_golden_reference(golden_dir):
    """generate_LRP_last_layer / full_lrp / attn_last_layer / rollout / attn_gradcam vs the reference's stored fp32
    outputs (NaN pattern included) and the fp64 oracle."""
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    g = np.load(os.path.join(golden_dir, "bert_generators.npz"))
    params, heads = obert.init_params(seed=int(g["param_seed"]), vocab=100, max_pos=32, dim=64, depth=3, heads=4,
                                      inter=128, rand_affine=True)
    model = make_model(params, heads, **TINY)
    gen = Generator(model)
    ids, mask = T(g["ids"]), T(g["mask"])
    p64 = {k: v.double() for k, v in params.items()}
    tol = {"LRP_last_layer": 2e-2, "full_lrp": 2e-2, "attn_last_layer": 1e-5, "rollout": 1e-5, "attn_gradcam": 2e-3}
    for key in [k for k in g.files if k.startswith("f32.")]:
        _, s, which, tag = key.split(".")
        s = int(s[1:])
        kw = {"start_layer": int(tag[2:])} if tag.startswith("sl") else ({} if tag == "argmax" else {"index": int(tag[5:])})
        out = getattr(gen, "generate_" + which)(ids[s:s + 1].cuda(), mask[s:s + 1].cuda(), **kw)
        ref = T(g[key])
        assert out.shape == ref.shape == (1, 24), key
        assert torch.equal(torch.isnan(out.cpu()), torch.isnan(ref)), key
        if torch.isnan(ref).any():
            continue
        ref64 = obert.generate(p64, ids[s:s + 1], mask[s:s + 1], heads, which, **kw)
        assert rel(out, ref64) < tol[which], "%s rel=%g" % (key, rel(out, ref64))
    # a batch is a set of independent sequences
    both = gen.generate_full_lrp(ids.cuda(), mask.cuda())
    one = gen.generate_full_lrp(ids[1:2].cuda(), mask[1:2].cuda())
    assert torch.allclose(both[1:2], one, rtol=1e-4, atol=1e-10)
