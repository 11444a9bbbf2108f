"""GPU: every explanation entry point and engine mode at tensor-core width, under every kernel selection, against fp64.

The tiny golden models (D = 64, dh = 16) satisfy no tensor-core predicate (Linear / z+ kernels need widths that are
multiples of 128, attention kernels dh in {32, 64}), so there every method runs the fp32 SIMT kernels only.  Here the
models are of real width with 3 blocks, so that ``last_layer``, ``second_layer`` and ``start_layer`` 0 / 1 are four
different relprop stops, and conditioned (``oracle/conditioned.py``) so that the fp32 CPU oracle agrees with the fp64
oracle to < 1e-4 of the map maximum (BERT maps: of the map range over the real tokens), checked per case (the regime
gate of ``test_gpu_parity_full.py``):

- ViT: D = 768, 12 heads, MLP 3072, 224/16 images (N = 197), 100 classes, batch 2; its distilled variant (N = 198);
- BERT: hidden 768, 12 heads, intermediate 3072, S = 130 (two row tiles, the second ragged), batch 3, one row padded
  from the middle;
- mlp_ratio < 1.5 (ViT D = 256 with MLP 256 and 128, BERT hidden 256 / intermediate 256), where the scratch the engines
  lend to the fp16 backward split and to the z+ rules' |x| is wider than M * F (tests/test_workspace_layout.py).

Entry points, each through its facade: ``LRP.generate_LRP`` (every method, ``is_ablation``, start_layer 0 / 1: the
KEEP_ALL_CAMS, cam-only-stop and RELPROP_TO_INPUT modes), ``Baselines`` (GRADIENTS_ONLY), ``ViT_orig_LRP`` (RULES_LRP),
the BERT ``Generator`` and ``model.relprop``.  Flag sets: 0, FLAG_ALL_FAST (51), FLAG_BENCH_DEFAULT (7475),
51 | ZPLUS_BF16 (115), 7475 | ZPLUS_R_F16 | BACKWARD_F16 (32051).

Bounds, relative to the tensor maximum: fp32 SIMT 2e-4; tensor-core sets 5e-3 (as test_gpu_parity_full.py); sets with
ZPLUS_BF16 2e-2 (not measured at this size: the 1.5e-2 unit bound of test_tc_bf16_second_contraction); maps of the
forward only (``last_layer_attn``, the baseline / BERT rollout, ``attn_last_layer``) 1e-5; the min-max normalised
``cam_attn`` / ``attn_gradcam`` 1e-3 absolute.  Class index bit-exact, NaN pattern identical, padded BERT tokens exactly
zero.  Measured worst case over every case of a model, on one H100 80GB HBM3 at a 400 W power limit:
  ViT-B width       SIMT 5.8e-6 | tensor cores 7.5e-4 | with ZPLUS_BF16 2.2e-4 | forward-only 9.7e-7
  DeiT distilled    SIMT 5.4e-6 | tensor cores 5.9e-4 | with ZPLUS_BF16 1.5e-4
  ViT_orig_LRP      SIMT 3.9e-5 | tensor cores 1.7e-3 | with ZPLUS_BF16 1.7e-3
  Baselines         forward-only 1.6e-6 | cam_attn 7.4e-4 absolute
  BERT-base width   SIMT 7.9e-6 | tensor cores 3.3e-4 | with ZPLUS_BF16 3.2e-4 | forward-only 4.8e-6 | attn_gradcam 2.6e-4
  D = 256           ViT MLP 256: 6.4e-4, MLP 128: 5.5e-4, BERT intermediate 256: 1.0e-3 (tensor-core sets)
"""
import functools

import pytest
import torch

from oracle import bert as obert
from oracle import conditioned
from oracle import cpu as ocpu
from oracle import vit as ovit
from transformer_explainability_b200 import _lib

pytestmark = pytest.mark.gpu

FLAG_SETS = [0, _lib.FLAG_ALL_FAST, _lib.FLAG_BENCH_DEFAULT, _lib.FLAG_ALL_FAST | _lib.FLAG_ZPLUS_BF16,
             _lib.FLAG_BENCH_DEFAULT | _lib.FLAG_ZPLUS_R_F16 | _lib.FLAG_BACKWARD_F16]
NARROW_FLAG_SETS = [_lib.FLAG_ALL_FAST, _lib.FLAG_BENCH_DEFAULT | _lib.FLAG_BACKWARD_F16]
FWD_TOL, NORM_TOL, GATE = 1e-5, 1e-3, 1e-4
# q / k / v bias offset of the conditioned ViTs: the default 4 makes the softmax inputs so large that the fp32 forward alone
# is 1e-5 off fp64 (last_layer_attn), the forward-only bound; 1 keeps Q K^T > 0 and leaves it at 1e-6
VIT_C_QKV = 1.0


def tol(flags):
    if flags & _lib.FLAG_ZPLUS_BF16:
        return 2e-2
    return 5e-3 if flags & _lib.FLAG_TENSOR_CORES else 2e-4


def rel(a, b):
    b = torch.as_tensor(b).double().cpu()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def range_rel(a, b, live):
    """error over the real tokens relative to the reference's range there (the row-normalised BERT maps are flat)"""
    a, b = a.double().cpu()[live], torch.as_tensor(b).double().cpu()[live]
    return ((a - b).abs().max() / (b.max() - b.min()).clamp_min(1e-300)).item()


WORST = {}


def record(model, what, flags, err, bound):
    print("%s %s flags %d: %.1e (bound %.0e)" % (model, what, flags, err, bound))
    key = (model, bound)
    WORST[key] = max(WORST.get(key, 0.0), err)
    assert err < bound, "%s %s flags %d: %g >= %g" % (model, what, flags, err, bound)


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for (model, bound), err in sorted(WORST.items()):
        print("worst %s, bound %.0e: %.1e" % (model, bound, err))


# ---- ViT ------------------------------------------------------------------------------------------------------------
VIT_CASES = [("transformer_attribution", dict(start_layer=0)), ("transformer_attribution", dict(start_layer=1)),
             ("grad", {}), ("rollout", dict(start_layer=0)), ("rollout", dict(start_layer=1)), ("full", {}),
             ("last_layer", {}), ("last_layer", dict(is_ablation=True)), ("last_layer_attn", {}),
             ("second_layer", {}), ("second_layer", dict(is_ablation=True))]
DEIT_CASES = [("transformer_attribution", dict(start_layer=0)), ("full", {}), ("rollout", dict(start_layer=0)),
              ("last_layer", dict(is_ablation=True))]
ORIG_CASES = [("grad", {}), ("full", {}), ("last_layer", {}), ("rollout", dict(start_layer=0))]
NARROW_VIT_CASES = [("transformer_attribution", dict(start_layer=0)), ("full", {})]


def _case_id(method, kw):
    return method + "".join(".%s=%s" % kv for kv in sorted(kw.items()))


def _vit_setup(name, seed, xseed, cases, variant="ours", n=2, **over):
    params, heads = ovit.init_params(name, seed=seed, rand_affine=True, depth=3, classes=100, **over)
    params = conditioned.condition_vit(params, c_qkv=VIT_C_QKV)
    x = torch.randn(n, 3, 224, 224, generator=torch.Generator().manual_seed(xseed))
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    refs = {}
    for method, kw in cases:
        ref, idx = ovit.explain_method(p64, x.double(), heads, method, variant=variant, **kw)
        ref32, _ = ovit.explain_method(params, x, heads, method, variant=variant, **kw)
        refs[_case_id(method, kw)] = (ref, idx, rel(ref32, ref))
    return dict(params=params, heads=heads, x=x, refs=refs, cases=cases)


@pytest.fixture(scope="module")
def vit_b():
    return _vit_setup("vit_base_patch16_224", seed=11, xseed=12, cases=VIT_CASES)


@pytest.fixture(scope="module")
def deit():
    return _vit_setup("deit_base_distilled_patch16_224", seed=13, xseed=14, cases=DEIT_CASES)


@pytest.fixture(scope="module")
def vit_orig():
    return _vit_setup("vit_base_patch16_224", seed=15, xseed=16, cases=ORIG_CASES, variant="lrp")


def _vit_model(setup, module="ViT_LRP", **kw):
    import importlib
    mod = importlib.import_module("transformer_explainability_b200.baselines.ViT." + module)
    p = setup["params"]
    D = p["cls_token"].shape[-1]
    mlp = p["blocks.0.mlp.fc1.weight"].shape[0]
    m = mod.VisionTransformer(img_size=224, patch_size=16, embed_dim=D, depth=3, num_heads=setup["heads"],
                              mlp_ratio=mlp / D, qkv_bias=True, num_classes=100, **kw)
    m.load_state_dict(p)
    return m.cuda().eval()


def _run_vit_methods(tag, setup, model, flag_sets):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    lrp = LRP(model)
    x = setup["x"].cuda()
    for method, kw in setup["cases"]:
        assert setup["refs"][_case_id(method, kw)][2] < GATE, \
            "regime is not conditioned for %s %s: fp32 oracle vs fp64 oracle %g" % (tag, method, setup["refs"][_case_id(method, kw)][2])
    for flags in flag_sets:
        model.engine_flags = flags
        for method, kw in setup["cases"]:
            ref, ridx, _ = setup["refs"][_case_id(method, kw)]
            out = lrp.generate_LRP(x, method=method, **kw)
            torch.cuda.synchronize()
            assert out.shape == ref.shape
            assert torch.equal(model.engine().tensor("logits").argmax(-1).cpu(), ridx), "%s %s: class index" % (tag, method)
            bound = FWD_TOL if method == "last_layer_attn" else tol(flags)
            record(tag, _case_id(method, kw), flags, rel(out, ref), bound)


def _batched_equals_single(out, one, s):
    scale = out.abs().max().item()
    assert torch.allclose(one[0], out[s], rtol=1e-5, atol=1e-6 * scale), "batched call differs from the per-sample call"


def _pixel_conservation(model, prefix):
    """relprop_pixels: the pixel relevance of each sample sums to the relevance of its patch tokens (the z^B rule
    conserves; Rtok, the tokens' share of self.add's relevance, is left in tmp_d2)"""
    eng = model.engine()
    pc = eng.relprop_pixels(per_channel=True)
    rtok = eng.tensor("tmp_d2")[:, prefix:].double().cpu()
    pix = pc.double().cpu().sum(dim=(1, 2, 3))
    assert ((pix - rtok.sum(dim=(1, 2))).abs() < 1e-3 * rtok.abs().sum(dim=(1, 2))).all(), (pix, rtok.sum(dim=(1, 2)))


def test_vit_every_method_every_flag_set(vit_b):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    model = _vit_model(vit_b)
    _run_vit_methods("vit-b3", vit_b, model, FLAG_SETS)
    # batch = independent B=1 explanations, one method per engine mode, at the benched selection
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT
    lrp = LRP(model)
    x = vit_b["x"].cuda()
    for method, kw in [("rollout", {}), ("last_layer", {}), ("second_layer", dict(is_ablation=True)), ("full", {})]:
        out = lrp.generate_LRP(x, method=method, **kw)
        for s in range(x.shape[0]):
            _batched_equals_single(out, lrp.generate_LRP(x[s:s + 1], method=method, **kw), s)
    model(x)
    _pixel_conservation(model, 1)


def test_deit_distilled_methods_and_pixel_path(deit):
    model = _vit_model(deit, distilled=True)
    _run_vit_methods("deit-b3", deit, model, FLAG_SETS)
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT
    model(deit["x"].cuda())
    _pixel_conservation(model, 2)


def test_vit_orig_lrp_rules(vit_orig):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    model = _vit_model(vit_orig, module="ViT_orig_LRP")
    _run_vit_methods("vit-orig-lrp", vit_orig, model, FLAG_SETS)
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT
    lrp = LRP(model)
    x = vit_orig["x"].cuda()
    out = lrp.generate_LRP(x, method="grad")
    for s in range(x.shape[0]):
        _batched_equals_single(out, lrp.generate_LRP(x[s:s + 1], method="grad"), s)


@pytest.fixture(scope="module")
def vit_new():
    params, heads = ovit.init_params("vit_base_patch16_224", seed=17, rand_affine=True, depth=3, classes=100)
    params = conditioned.condition_vit(params, c_qkv=VIT_C_QKV)
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(18))
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    refs, gate = {}, {}
    for sl in (0, 1):
        refs[("rollout", sl)] = ovit.baseline_rollout(p64, x.double(), heads, start_layer=sl)
        gate[("rollout", sl)] = rel(ovit.baseline_rollout(params, x, heads, start_layer=sl), refs[("rollout", sl)])
    for index in (None, 7):
        refs[("cam_attn", index)] = ovit.baseline_cam_attn(p64, x.double(), heads, index=index)
        gate[("cam_attn", index)] = abs_err(ovit.baseline_cam_attn(params, x, heads, index=index)[0],
                                            refs[("cam_attn", index)][0])
    return dict(params=params, heads=heads, x=x, refs=refs, gate=gate)


def test_vit_baselines(vit_new):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import Baselines
    model = _vit_model(vit_new, module="ViT_new", norm_layer=functools.partial(torch.nn.LayerNorm, eps=1e-6))
    base = Baselines(model)
    x = vit_new["x"].cuda()
    for key, e in vit_new["gate"].items():
        assert e < GATE, "regime is not conditioned for the ViT baseline %s: fp32 oracle vs fp64 oracle %g" % (key, e)
    for flags in FLAG_SETS:
        model.engine_flags = flags
        for sl in (0, 1):
            record("vit-new", "rollout.start_layer=%d" % sl, flags, rel(base.generate_rollout(x, start_layer=sl),
                                                                           vit_new["refs"][("rollout", sl)]), FWD_TOL)
        for index in (None, 7):
            ref, ridx = vit_new["refs"][("cam_attn", index)]
            out = base.generate_cam_attn(x, index=index)
            torch.cuda.synchronize()
            if index is None:
                assert torch.equal(model.engine().tensor("logits").argmax(-1).cpu(), ridx)
            assert out.shape == ref.shape
            assert torch.equal(torch.isnan(out.cpu()), torch.isnan(ref)), "NaN pattern of cam_attn differs"
            record("vit-new", "cam_attn.index=%s" % index, flags, abs_err(out, ref), NORM_TOL)
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT
    out = base.generate_cam_attn(x, index=7)
    for s in range(x.shape[0]):
        one = base.generate_cam_attn(x[s:s + 1], index=7)
        assert torch.allclose(one, out[s], rtol=1e-5, atol=1e-6, equal_nan=True)


# ---- BERT -----------------------------------------------------------------------------------------------------------
BERT_GENERATORS = [("LRP", dict(start_layer=0)), ("LRP", dict(start_layer=1)), ("LRP_last_layer", {}),
                   ("full_lrp", {}), ("attn_last_layer", {}), ("rollout", dict(start_layer=0)), ("attn_gradcam", {})]
BERT_FORWARD_ONLY = ("attn_last_layer", "rollout")


def _bert_setup(seed, dim, heads, inter, cases, n=3, seq=130, c_qkv=3.0):
    params, heads = obert.init_params(seed=seed, vocab=1000, max_pos=512, dim=dim, depth=3, heads=heads, inter=inter,
                                      rand_affine=True)
    params = conditioned.condition_bert(params, c_qkv=c_qkv)
    g = torch.Generator().manual_seed(seed + 1)
    ids = torch.randint(5, 1000, (n, seq), generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    mask = torch.ones(n, seq, dtype=torch.long)
    pad = seq // 2
    mask[1, pad:] = 0                                              # sample 1 is padded from the middle on
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    refs = {}
    for which, kw in cases:
        if which == "LRP":
            ref, idx = obert.explain(p64, ids, mask, heads, **kw)
            ref32, _ = obert.explain(params, ids, mask, heads, **kw)
        else:
            ref = obert.generate(p64, ids, mask, heads, which, **kw)
            ref32 = obert.generate(params, ids, mask, heads, which, **kw)
            idx = None
        refs[_case_id(which, kw)] = (ref, idx, ref32)
    # model.relprop: relevance at the encoder input [B,S,D]
    refs["relprop"] = (_bert_relprop(p64, ids, mask, heads), None, _bert_relprop(params, ids, mask, heads))
    return dict(params=params, heads=heads, ids=ids, mask=mask, pad=pad, refs=refs, cases=cases,
                cfg=dict(hidden_size=dim, num_hidden_layers=3, intermediate_size=inter, vocab_size=1000,
                         max_position_embeddings=512))


def _bert_relprop(params, ids, mask, heads):
    with torch.enable_grad():
        logits, cache = obert.forward(params, ids, mask, heads)
    seed = torch.zeros_like(logits)
    seed[torch.arange(logits.shape[0]), logits.argmax(-1)] = 1
    with torch.no_grad():
        cd = {"dims": cache["dims"], "ext_mask": cache["ext_mask"], "h_last": cache["h_last"].detach(),
              "pooled": cache["pooled"].detach(), "layers": [{k: v.detach() for k, v in c.items()} for c in cache["layers"]]}
        _, r = obert.relprop(params, cd, seed.detach(), lowest=0, to_input=True)
    return r


def abs_err(out, ref):
    """max absolute error over the entries the reference does not leave NaN (min-max normalised maps)"""
    ref = torch.as_tensor(ref).double().cpu()
    ok = ~torch.isnan(ref)
    return (out.double().cpu() - ref).abs()[ok].max().item() if ok.any() else 0.0


def _gate_bert(setup, live):
    for key, (ref, _, ref32) in setup["refs"].items():
        if key.startswith("attn_gradcam"):
            e = abs_err(ref32, ref)
        elif ref.dim() == 2:
            e = max(range_rel(ref32[s], ref[s], live[s]) for s in range(ref.shape[0]))
        else:
            e = rel(ref32, ref)
        assert e < GATE, "regime is not conditioned for bert %s: fp32 oracle vs fp64 oracle %g" % (key, e)


def _run_bert(tag, setup, flag_sets):
    from test_gpu_bert import make_model
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    model = make_model(setup["params"], setup["heads"], **setup["cfg"])
    gen = Generator(model)
    ids, mask, pad = setup["ids"].cuda(), setup["mask"].cuda(), setup["pad"]
    live = setup["mask"].bool()
    _gate_bert(setup, live)
    for flags in flag_sets:
        model.engine_flags = flags
        for which, kw in setup["cases"]:
            ref, ridx, _ = setup["refs"][_case_id(which, kw)]
            out = getattr(gen, "generate_" + which)(ids, mask, **kw)
            torch.cuda.synchronize()
            assert out.shape == ref.shape
            if ridx is not None:
                assert torch.equal(model.engine().tensor("logits").argmax(-1).cpu(), ridx), "%s %s: class index" % (tag, which)
            nan = torch.isnan(ref)
            assert torch.equal(torch.isnan(out.cpu()), nan), "%s %s: NaN pattern" % (tag, which)
            if not nan[1].any():                                   # an all-zero GradCAM normalises to NaN
                assert float(out[1, pad:].abs().max()) == 0.0, "%s %s: padded tokens must get exactly zero" % (tag, which)
            if which == "attn_gradcam":
                record(tag, _case_id(which, kw), flags, abs_err(out, ref), NORM_TOL)
                continue
            bound = FWD_TOL if which in BERT_FORWARD_ONLY else tol(flags)
            record(tag, _case_id(which, kw), flags, rel(out, ref), bound)
            print("    %s of the range over the real tokens: %.1e" % (
                _case_id(which, kw), max(range_rel(out[s], ref[s], live[s]) for s in range(ref.shape[0]))))
        logits = model(ids, mask)[0]
        oh = torch.zeros_like(logits)
        oh[torch.arange(logits.shape[0]), logits.argmax(-1)] = 1
        r_in = model.relprop(oh, alpha=1)
        torch.cuda.synchronize()
        ref = setup["refs"]["relprop"][0]
        assert r_in.shape == ref.shape
        assert float(r_in[1, pad:].abs().max()) == 0.0
        record(tag, "relprop", flags, rel(r_in, ref), tol(flags))
    return model, gen


@pytest.fixture(scope="module")
def bert_b():
    return _bert_setup(seed=22, dim=768, heads=12, inter=3072, cases=BERT_GENERATORS)


def test_bert_every_generator_every_flag_set(bert_b):
    model, gen = _run_bert("bert-b3", bert_b, FLAG_SETS)
    model.engine_flags = _lib.FLAG_BENCH_DEFAULT
    ids, mask = bert_b["ids"].cuda(), bert_b["mask"].cuda()
    for which, kw in [("full_lrp", {}), ("attn_gradcam", {}), ("LRP", dict(start_layer=1)), ("LRP_last_layer", {})]:
        out = getattr(gen, "generate_" + which)(ids, mask, **kw)
        for s in range(ids.shape[0]):
            one = getattr(gen, "generate_" + which)(ids[s:s + 1], mask[s:s + 1], **kw)
            _batched_equals_single(out, one, s)


# ---- mlp_ratio < 1.5: the lent scratch regions are wider than M * F ------------------------------------------------------
@pytest.mark.parametrize("mlp", [256, 128])
def test_vit_narrow_mlp(mlp):
    setup = _vit_setup("vit_base_patch16_224", seed=31 + mlp, xseed=32, cases=NARROW_VIT_CASES, dim=256, heads=4, mlp=mlp)
    model = _vit_model(setup)
    _run_vit_methods("vit-d256-mlp%d" % mlp, setup, model, NARROW_FLAG_SETS)


def test_bert_narrow_intermediate():
    setup = _bert_setup(seed=41, dim=256, heads=4, inter=256, cases=[("LRP", dict(start_layer=0)), ("full_lrp", {})])
    _run_bert("bert-d256-f256", setup, NARROW_FLAG_SETS)
