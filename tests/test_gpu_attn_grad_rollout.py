"""GPU: the gradient-weighted attention rollout (TE_FLAG_ATTN_GRAD_ROLLOUT) of the ViT / DeiT / BERT engines.

- Tiny golden models against the fixture's fp64 maps (``tests/golden/attn_grad_rollout.npz``: the reference's own attention
  maps and gradients, the rule applied in fp64).
- Full size on random-init weights (no conditioning: the map is built from clamped products and non-negative sums, no
  safe_divide): ViT-B/16 (``oracle.vit.init_params(seed=0)``, the weights of ``vit_base.npz``), DeiT-B-distilled and
  BERT-base at S = 130, batch 3 with one row padded from the middle, explicit class indices, against the fp64 oracle at
  flag sets 0, 51, 7475 and 32051 and start_layer 0, 1 and L-1.  Bounds relative to the map maximum: 2e-4 SIMT, 5e-3 for
  the tensor-core sets (those of test_gpu_methods_tc.py), and the same regime gate: the fp32 oracle within 1e-4 of fp64.
- The fused row kernel and the composed rollout agree to 1e-5 of the largest entry of row 0 (R[0, 0], which carries the
  rollout's rounding; the map leaves that column out and is ~1e-2 of it on random-init weights); the engine equals ``ops.attribution_rollout`` on its own
  ``attn_grad`` / ``attn`` taps bit for bit at the matching rollout selection; the rule-library bits change no bit.
- Batched equals per-sample, chunked equals unchunked, padded BERT entries are exactly 0 and the real tokens match the
  unpadded run; poisoned workspaces / outputs (test_gpu_poison.py's allocator) give identical bits; attn_cam keeps a
  poison written before ``attribute`` (no relprop ran) and no forward tap changes; CUDA-graph replay is bit-identical.
- Rejected flag combinations and alpha != 1 return errors; each evaluation command runs the method end to end.
"""
import os

import numpy as np
import pytest
import torch

from oracle import attn_grad_rollout as agr
from oracle import bert as obert
from oracle import cpu as ocpu
from oracle import vit as ovit
from transformer_explainability_b200 import _lib

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
AGR = _lib.FLAG_ATTN_GRAD_ROLLOUT
FLAG_SETS = [0, _lib.FLAG_ALL_FAST, _lib.FLAG_BENCH_DEFAULT,
             _lib.FLAG_BENCH_DEFAULT | _lib.FLAG_ZPLUS_R_F16 | _lib.FLAG_BACKWARD_F16]
GATE = 1e-4


def tol(flags):
    return 5e-3 if flags & _lib.FLAG_TENSOR_CORES else 2e-4


def rel(a, b):
    b = torch.as_tensor(b).double().cpu()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def _vit_facade(params, heads, img, patch, depth, classes, module="ViT_LRP", flags=0):
    import functools
    import importlib
    import torch.nn as nn
    mod = importlib.import_module("transformer_explainability_b200.baselines.ViT." + module)
    D = params["cls_token"].shape[-1]
    mlp = params["blocks.0.mlp.fc1.weight"].shape[0]
    kw = {"distilled": True} if "dist_token" in params else {}
    if module == "ViT_new":                      # every LayerNorm at 1e-6, as the ViT_new factories
        kw["norm_layer"] = functools.partial(nn.LayerNorm, eps=1e-6)
    m = mod.VisionTransformer(img_size=img, patch_size=patch, embed_dim=D, depth=depth, num_heads=heads,
                              mlp_ratio=mlp / D, qkv_bias=True, num_classes=classes, **kw)
    m.load_state_dict(params)
    m.engine_flags = flags
    return m.cuda().eval()


def _bert_facade(params, heads, cls_lrp=False, **cfg):
    from transformers import BertConfig
    if cls_lrp:
        from transformer_explainability_b200.BERT_explainability.modules.BERT.BERT_cls_lrp import \
            BertForSequenceClassification
    else:
        from transformer_explainability_b200.BERT_explainability.modules.BERT.BertForSequenceClassification import \
            BertForSequenceClassification
    m = BertForSequenceClassification(BertConfig(num_attention_heads=heads, num_labels=2, **cfg))
    res = m.load_state_dict({k: v.float() for k, v in params.items()}, strict=False)
    assert not res.unexpected_keys
    return m.cuda().eval()


# ---- tiny golden models ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def z():
    return np.load(os.path.join(HERE, "golden", "attn_grad_rollout.npz"))


@pytest.mark.parametrize("model", ["vit", "deit"])
@pytest.mark.parametrize("module", ["ViT_LRP", "ViT_orig_LRP", "ViT_new"])
def test_tiny_vit_against_the_fixture(z, model, module):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    if model == "deit" and module != "ViT_LRP":
        pytest.skip("the distilled variant is a ViT_LRP extension")
    p, h = ovit.init_params("vit_tiny_test", seed=int(z[model + ".param_seed"]), rand_affine=True,
                            distilled=(model == "deit"))
    m = _vit_facade(p, h, 32, 8, 3, 10, module=module)
    x = torch.from_numpy(z["x"]).cuda()
    refs = {}
    if module == "ViT_new":
        # ViT_new's final LayerNorm epsilon (1e-6) is not the fixture model's (1e-5): its reference is the fp64 oracle
        for sl in z["start_layers"]:
            r, i = agr.explain_vit({k: v.double() for k, v in p.items()}, x.cpu().double(), h, start_layer=int(sl),
                                   norm_eps=1e-6)
            refs[int(sl)] = (r, i)
    for flags in (0, _lib.FLAG_BENCH_DEFAULT):
        m.engine_flags = flags
        for sl in z["start_layers"]:
            maps = LRP(m).generate_attn_grad_rollout(x, start_layer=int(sl))
            assert maps.shape == (2, 16)
            idx = m.engine().tensor("logits").argmax(-1).cpu()
            for s in range(2):
                key = "%s.f64.s%d" % (model, s)
                if refs:
                    want, widx = refs[int(sl)][0][s], int(refs[int(sl)][1][s])
                else:
                    want, widx = z["%s.map.sl%d" % (key, sl)][0], int(z[key + ".index"])
                assert int(idx[s]) == widx
                err = rel(maps[s], want)
                print("tiny %s %s flags %d sl %d: %.1e" % (model, module, flags, sl, err))
                assert err < tol(flags), (key, flags, int(sl), err)


@pytest.mark.parametrize("cls_lrp", [False, True])
def test_tiny_bert_against_the_fixture(z, cls_lrp):
    from test_gpu_bert import TINY
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    p, h = obert.init_params(seed=int(z["bert.param_seed"]), vocab=100, max_pos=32, dim=64, depth=3, heads=4, inter=128,
                             rand_affine=True)
    m = _bert_facade(p, h, cls_lrp=cls_lrp, **TINY)
    ids, mask = torch.from_numpy(z["ids"]).cuda(), torch.from_numpy(z["mask"]).cuda()
    for sl in z["start_layers"]:
        maps = Generator(m).generate_attn_grad_rollout(ids, mask, start_layer=int(sl))
        assert maps.shape == ids.shape
        for s in range(2):
            key = "bert.f64.s%d" % s
            want = z["%s.map.sl%d" % (key, sl)][0]
            assert int(m.engine().tensor("logits").argmax(-1)[s]) == int(z[key + ".index"])
            assert (maps[s].cpu()[torch.from_numpy(want) == 0] == 0).all()
            assert rel(maps[s], want) < 2e-4, (key, int(sl))


# ---- full size, random-init weights ---------------------------------------------------------------------------------------
def _vit_case(name, n=2):
    params, heads = ovit.init_params(name, seed=0)
    x = torch.randn(n, 3, 224, 224, generator=torch.Generator().manual_seed(100))
    index = torch.tensor([3, 517][:n])
    ocpu.set_torch_threads()
    a64, g64, _ = agr.vit_taps({k: v.double() for k, v in params.items()}, x.double(), heads, index)
    a32, g32, _ = agr.vit_taps(params, x, heads, index)
    L = len(a64)
    prefix = 2 if "dist_token" in params else 1
    refs = {}
    for sl in (0, 1, L - 1):
        r64 = agr.vit_map(a64, g64, sl, prefix)
        refs[sl] = (r64, rel(agr.vit_map(a32, g32, sl, prefix), r64))
    return dict(params=params, heads=heads, x=x, index=index, refs=refs, L=L, prefix=prefix)


@pytest.fixture(scope="module")
def vit_b():
    return _vit_case("vit_base_patch16_224")


@pytest.fixture(scope="module")
def deit():
    return _vit_case("deit_base_distilled_patch16_224")


def _bert_inputs(n=3, S=130, vocab=30522):
    g = torch.Generator().manual_seed(31)
    ids = torch.randint(1000, vocab, (n, S), generator=g)
    mask = torch.ones(n, S, dtype=torch.long)
    mask[1, S // 2:] = 0
    return ids, mask


@pytest.fixture(scope="module")
def bert_b():
    params, heads = obert.init_params(seed=0)
    ids, mask = _bert_inputs()
    index = torch.tensor([1, 0, 1])
    ocpu.set_torch_threads()
    a64, g64, _ = agr.bert_taps({k: v.double() for k, v in params.items()}, ids, mask, heads, index)
    a32, g32, _ = agr.bert_taps(params, ids, mask, heads, index)
    L = len(a64)
    refs = {}
    for sl in (0, 1, L - 1):
        r64 = agr.bert_map(a64, g64, sl)
        refs[sl] = (r64, rel(agr.bert_map(a32, g32, sl), r64))
    return dict(params=params, heads=heads, ids=ids, mask=mask, index=index, refs=refs, L=L)


def _check_regime(tag, refs):
    for sl, (_, gate) in refs.items():
        print("%s sl %d: fp32 oracle vs fp64 %.1e (gate %.0e)" % (tag, sl, gate, GATE))
        assert gate < GATE, "%s start_layer %d: fp32 oracle vs fp64 oracle %g" % (tag, sl, gate)


def _layer_stack(eng, name, L):
    """[L, B, H, N, NP] copy of a per-layer workspace tensor, pad columns included (the engine's own layout)"""
    v0 = eng.tensor(name, 0)
    ls = eng.tensor(name, 1).storage_offset() - v0.storage_offset()
    B, H, N, _ = v0.shape
    NP = v0.stride(2)
    return torch.as_strided(eng._ws, (L, B, H, N, NP), (ls, v0.stride(0), v0.stride(1), NP, 1),
                            v0.storage_offset()).contiguous()


@pytest.mark.parametrize("case", ["vit_b", "deit"])
def test_full_size_vit_against_fp64(case, request):
    from transformer_explainability_b200 import ops
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    c = request.getfixturevalue(case)
    _check_regime(case, c["refs"])
    m = _vit_facade(c["params"], c["heads"], 224, 16, c["L"], 1000)
    lrp, x, idx = LRP(m), c["x"].cuda(), c["index"].cuda()
    worst = {}
    for flags in FLAG_SETS:
        m.engine_flags = flags
        for sl, (ref, _) in c["refs"].items():
            maps = lrp.generate_attn_grad_rollout(x, index=idx, start_layer=sl)
            torch.cuda.synchronize()
            assert maps.shape == ref.shape
            err = rel(maps, ref)
            worst[tol(flags)] = max(worst.get(tol(flags), 0.0), err)
            print("%s flags %d sl %d: %.1e (bound %.0e)" % (case, flags, sl, err, tol(flags)))
            assert err < tol(flags), (case, flags, sl, err)
            # the engine's rollout equals ops.attribution_rollout on its own taps at the same selection, bit for bit
            eng = m.engine()
            g, a = _layer_stack(eng, "attn_grad", c["L"]), _layer_stack(eng, "attn", c["L"])
            _, row0 = ops.attribution_rollout(g, a, start_layer=sl, fused=bool(flags & _lib.FLAG_ROLLOUT_FUSED),
                                              want_joint=False)
            assert torch.equal(maps, row0[:, c["prefix"]:]), (case, flags, sl)
            # the other rollout selection on the same taps, relative to the largest entry of row 0: R[0, 0] >= 1 carries
            # the rollout's rounding, and the map leaves that column out (its maximum is ~1e-2 on random-init weights)
            _, other = ops.attribution_rollout(g, a, start_layer=sl, fused=not flags & _lib.FLAG_ROLLOUT_FUSED,
                                               want_joint=False)
            sel = ((other - row0).abs().max() / row0.abs().max()).item()
            worst["selection"] = max(worst.get("selection", 0.0), sel)
            assert sel < 1e-5, (case, flags, sl, sel)
    print("MEASURED %s worst: %s" % (case, {k: "%.1e" % v for k, v in worst.items()}))
    # fused and composed rollout through the engine itself (the same taps: ROLLOUT_FUSED selects nothing else)
    m.engine_flags = _lib.FLAG_BENCH_DEFAULT
    fused = lrp.generate_attn_grad_rollout(x, index=idx).clone()
    m.engine_flags = _lib.FLAG_BENCH_DEFAULT & ~_lib.FLAG_ROLLOUT_FUSED
    composed = lrp.generate_attn_grad_rollout(x, index=idx)
    eng = m.engine()
    _, row0 = ops.attribution_rollout(_layer_stack(eng, "attn_grad", c["L"]), _layer_stack(eng, "attn", c["L"]),
                                      want_joint=False)
    assert ((composed - fused).abs().max() / row0.abs().max()).item() < 1e-5


def test_full_size_bert_against_fp64(bert_b):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    c = bert_b
    _check_regime("bert-b", c["refs"])
    m = _bert_facade(c["params"], c["heads"])
    gen, ids, mask, idx = Generator(m), c["ids"].cuda(), c["mask"].cuda(), c["index"].cuda()
    pad = c["mask"] == 0
    for flags in FLAG_SETS:
        m.engine_flags = flags
        for sl, (ref, _) in c["refs"].items():
            maps = gen.generate_attn_grad_rollout(ids, mask, index=idx, start_layer=sl)
            torch.cuda.synchronize()
            err = rel(maps, ref)
            print("bert-b flags %d sl %d: %.1e (bound %.0e)" % (flags, sl, err, tol(flags)))
            assert err < tol(flags), (flags, sl, err)
            mc = maps.cpu()
            assert (mc[pad] == 0).all() and (mc[:, 0] == 0).all(), "padded entries / element 0 are not exactly 0"
        # the padded row against its unpadded run: real tokens within the padding bound of test_gpu_eraser.py
        n = int(c["mask"][1].sum())
        full = gen.generate_attn_grad_rollout(ids, mask, index=idx)
        one = gen.generate_attn_grad_rollout(ids[1:2, :n], mask[1:2, :n], index=idx[1:2])
        assert rel(full[1:2, :n], one) < tol(flags)


# ---- invariances, poison, graph replay, errors -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_vit():
    """ViT-B width, 3 blocks: every kernel selection of the full model at a fraction of the cost"""
    p, h = ovit.init_params("vit_base_patch16_224", seed=5, depth=3, classes=100)
    m = _vit_facade(p, h, 224, 16, 3, 100, flags=_lib.FLAG_BENCH_DEFAULT)
    x = torch.randn(3, 3, 224, 224, generator=torch.Generator().manual_seed(6)).cuda()
    return m, x


def test_rule_library_bits_change_nothing(small_vit):
    m, x = small_vit
    eng = m.engine()
    base, i0 = eng.explain(x, flags=_lib.FLAG_BENCH_DEFAULT | AGR)
    lrp, i1 = eng.explain(x, flags=_lib.FLAG_BENCH_DEFAULT | AGR | _lib.FLAG_RULES_LRP | _lib.FLAG_RULES_LRP_TC)
    assert torch.equal(base, lrp) and torch.equal(i0, i1)
    other, _ = eng.explain(x, flags=_lib.FLAG_BENCH_DEFAULT | AGR | _lib.FLAG_ZPLUS_BF16 | _lib.FLAG_ZPLUS_R_F16)
    assert torch.equal(base, other)


@pytest.mark.parametrize("flags", [0, _lib.FLAG_BENCH_DEFAULT])
def test_batched_and_chunked(small_vit, flags):
    m, x = small_vit
    eng = m.engine()
    full, idx = eng.explain(x, flags=flags | AGR)
    chunked, idx2 = eng.explain(x, flags=flags | AGR, chunk=1)
    assert torch.equal(idx, idx2)
    scale = full.abs().max().item()
    assert torch.allclose(chunked, full, rtol=1e-5, atol=1e-6 * scale)
    for s in range(x.shape[0]):
        one, _ = eng.explain(x[s:s + 1], flags=flags | AGR)
        assert torch.allclose(one[0], full[s], rtol=1e-5, atol=1e-6 * scale)


def test_no_relprop_and_no_forward_tap_changes(small_vit):
    m, x = small_vit
    eng = m.engine()
    fl = _lib.FLAG_BENCH_DEFAULT | AGR
    eng.forward(x, flags=fl)
    ref, _ = eng.attribute(flags=fl)
    eng.forward(x, flags=fl)
    L = 3
    taps = {"logits": eng.tensor("logits").clone()}
    for l in range(L):
        for name in ("attn", "x_in", "qkv"):
            taps["%s%d" % (name, l)] = eng.tensor(name, l).clone()
    cams = [eng.tensor("attn_cam", l) for l in range(L)]
    for c in cams:
        c.view(torch.int32).fill_(0x5A5A5A5A)
    out, _ = eng.attribute(flags=fl)
    assert torch.equal(out, ref)
    for c in cams:
        assert (c.contiguous().view(torch.int32) == 0x5A5A5A5A).all(), "attn_cam was written: the relprop ran"
    for k, v in taps.items():
        name, l = (k, None) if k == "logits" else (k.rstrip("0123456789"), int(k[len(k.rstrip("0123456789")):]))
        now = eng.tensor(name) if l is None else eng.tensor(name, l)
        assert torch.equal(now, v), "%s changed during attribute" % k


@pytest.mark.parametrize("flags", [0, _lib.FLAG_BENCH_DEFAULT | _lib.FLAG_ZPLUS_R_F16 | _lib.FLAG_BACKWARD_F16])
def test_poisoned_runs_are_bit_identical(small_vit, flags):
    from test_gpu_poison import EngineState, Findings, _poison_from, run_case
    m, x = small_vit
    eng = m.engine()
    found = Findings()
    idx = torch.tensor([7, 1, 42], dtype=torch.int32).cuda()
    for sl in (0, 2):
        def fn(pattern, sl=sl):
            eng.forward(x, flags=flags | AGR)
            _poison_from(eng, "tmp_d0", pattern)
            maps, cls = eng.attribute(index=idx, start_layer=sl, flags=flags | AGR)
            out = {"maps": maps, "index": cls, "logits": eng.tensor("logits")}
            out.update({"attn_grad%d" % l: eng.tensor("attn_grad", l) for l in range(sl, 3)})
            return out
        run_case(found, "vit-b3 flags %d sl %d" % (flags, sl), fn, before=EngineState(eng))
        run_case(found, "vit-b3 flags %d sl %d explain" % (flags, sl),
                 lambda pattern, sl=sl: eng.explain(x, index=idx, start_layer=sl, flags=flags | AGR),
                 before=EngineState(eng))
    found.check()


def test_graph_replay_is_bit_identical(small_vit):
    m, x = small_vit
    eng = m.engine()
    fl = _lib.FLAG_BENCH_DEFAULT | AGR
    ref, ridx = eng.explain(x, flags=fl, start_layer=1)
    for _ in range(2):
        maps, idx = eng.explain_graphed(x, flags=fl, start_layer=1)
        assert torch.equal(maps, ref) and torch.equal(idx, ridx)


def test_sharded_explain_passes_the_flag(small_vit):
    from transformer_explainability_b200 import parallel
    m, x = small_vit
    eng = m.engine()
    ref, _ = eng.explain(x, flags=eng.flags | AGR)
    eng.flags = m.engine_flags | AGR
    try:
        maps, _ = parallel.explain_sharded(eng, x)
        gmaps, _ = parallel.explain_sharded(eng, x, graph=True)
    finally:
        eng.flags = m.engine_flags
    assert torch.equal(maps, ref) and torch.equal(gmaps, ref)


def test_rejected_combinations(small_vit, z):
    from test_gpu_bert import TINY
    m, x = small_vit
    eng = m.engine()
    eng.forward(x)
    p, h = obert.init_params(seed=3, vocab=100, max_pos=32, dim=64, depth=3, heads=4, inter=128)
    beng = _bert_facade(p, h, **TINY).engine()
    beng.forward(torch.from_numpy(z["ids"]).cuda(), torch.from_numpy(z["mask"]).cuda())
    for e in (eng, beng):
        for bad in (_lib.FLAG_GRADIENTS_ONLY, _lib.FLAG_KEEP_ALL_CAMS, _lib.FLAG_RELPROP_TO_INPUT):
            with pytest.raises(_lib.TeError, match="does not combine") as ex:
                e.attribute(start_layer=0, flags=AGR | bad)
            assert ex.value.status == -1
        with pytest.raises(_lib.TeError, match="alpha must be 1") as ex:
            e.attribute(start_layer=0, flags=AGR, alpha=0.5)
        assert ex.value.status == -1
        e.attribute(start_layer=0, flags=AGR)                           # and the engine still works afterwards


# ---- the evaluation commands ---------------------------------------------------------------------------------------------------
def test_commands_run_the_method(small_vit, tmp_path):
    from transformer_explainability_b200 import hdf5_writer, segmentation, visualization
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    m, x = small_vit
    lrp = LRP(m)
    want = lrp.generate_attn_grad_rollout(x).clone()
    # segmentation: the map it thresholds
    assert torch.equal(segmentation.explain("attn_grad_rollout", x, lrp=lrp), want)
    # hdf5_writer: the heat maps written to results.hdf5 are those of the façade's maps
    imgs = torch.rand(3, 3, 224, 224, generator=torch.Generator().manual_seed(8))
    d = str(tmp_path / "visualizations" / "attn_grad_rollout" / "top" / "not_ablation")
    path = hdf5_writer.compute_saliency_and_save([(imgs, torch.tensor([0, 1, 2]))], d, "attn_grad_rollout", lrp=lrp,
                                                   backend="builtin")
    got = hdf5_writer.read_minimal_hdf5(path)
    heat = visualization.relevance_to_heatmap(lrp.generate_attn_grad_rollout(hdf5_writer.normalize(imgs.cuda())))
    assert np.array_equal(np.asarray(got["vis"]).reshape(3, -1), heat.reshape(3, -1).cpu().numpy())
    # visualization: overlays of the façade's maps
    ov = visualization.generate_visualizations(lrp, x, method="attn_grad_rollout")
    assert torch.equal(ov, visualization.render_overlays(x, visualization.relevance_to_heatmap(want)))
    one = visualization.generate_visualization(lrp, x[0], method="attn_grad_rollout")
    assert np.array_equal(one, visualization.render_overlays(
        x[:1], visualization.relevance_to_heatmap(lrp.generate_attn_grad_rollout(x[:1])))[0].cpu().numpy())


def test_eraser_runs_the_method():
    import functools
    from test_gpu_eraser import THRESHOLDS, _fixture
    from test_gpu_bert import make_model, TINY
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    g, docids, docs, anns, enc, te = _fixture()
    zz = np.load(os.path.join(HERE, "golden", "bert_tiny.npz"))
    params = {k[len("param."):]: torch.from_numpy(zz[k]) for k in zz.files if k.startswith("param.")}
    gen = Generator(make_model(params, int(zz["heads"]), **TINY)).generate_attn_grad_rollout
    classes = {"NEG": 0, "POS": 1}
    res = te.eraser_eval(gen, docs, anns, enc, classes, batch_size=4, iou_thresholds=THRESHOLDS, faithfulness=True,
                         soft_scores=True)
    one = te.eraser_eval(functools.partial(gen), docs, anns, enc, classes, batch_size=1, iou_thresholds=THRESHOLDS)
    assert res["docids"] == one["docids"] and "faithfulness" in res and "soft" in res
    # padded, length-sorted batches rank the words as the per-document runs do (up to rounding ties)
    same = np.mean([np.array_equal(a, b) for a, b in zip(res["order"], one["order"])])
    assert same >= 0.9, same
