"""GPU: the engines on the published small ViT / DeiT / BERT geometries, where kernel selection splits between the tensor
cores and SIMT inside one engine call, against fp64.

Both engines pick a kernel at every call site from shape predicates (te_tc_wgmma.cu, te_engine_util.h, te_rollout.cu):
forward / backward Linears on the tensor cores for K % 32 == 0 and N % 128 == 0 (the fp16 forms K % 64 == 0; the fp16-split
forward only when all four Linears of a block qualify and F >= D), the z+ / layers_lrp rules for in and out % 128 == 0, the
N x N attention contractions for dh in {32, 64}, the token reductions for dh == 64, the fused row rollout for
round_up(N, 4) <= 512 (otherwise the dense chain and extract_row_kernel).  At the widths of test_gpu_methods_tc.py every site
qualifies, on the tiny golden models none does.  Here (3 blocks, conditioned as in test_gpu_methods_tc.py, c_qkv = 1 for ViT;
ViT 224/16 unless stated, batch 2, 100 classes; BERT S = 130, batch 3, one row padded from the middle):

  vit-ti       D 192, H 3, MLP 768      fc1 forward / fc2 backward (K = 192) on the tensor cores, every other Linear and every
                                        z+ rule SIMT, no fp16-split forward at 7475, H = 3 in the fused row rollout
  vit-s        D 384, H 6, MLP 1536     every in-block site on the tensor cores, fp16-split forward on
  deit-s-dist  vit-s distilled (N = 198)
  vit-dh32     D 384, H 12, MLP 1536    N x N contractions at dh 32, token reductions SIMT
  vit-dh48     D 384, H 8, MLP 1536     all attention SIMT, Linears and z+ rules on the tensor cores
  vit-b-384    D 768, H 12, img 384     N = 577: maps from the dense rollout chain + extract_row_kernel
  bert-tiny    hidden 128, H 2, inter 512      one 128-column tile everywhere
  bert-minilm  hidden 384, H 12, inter 1536    dh 32 in the BERT engine
  bert-small   hidden 512, H 8, inter 2048     an all-tensor-core width

A kernel census (torch.profiler, kernel names reduced to families as tools/profile_step_kernels.py does) checks that each
geometry runs the mix it claims.  Flag sets 0, 51, 7475, 32051 (RULES_LRP_TC added for the layers_lrp cases).  Each case first
passes the regime gate: fp32 oracle within 1e-4 of fp64.  Bounds as in test_gpu_methods_tc.py: SIMT 2e-4, tensor-core sets
5e-3, forward-only maps 1e-5, min-max normalised maps 1e-3 absolute; per-layer taps as in test_gpu_engine_shapes.py
(probabilities 1e-5, attention gradients 1e-4, top attn_cam 5e-2), except that with TE_FLAG_BACKWARD_TF32 the attention
gradients and the normalised maps built from them take the single-pass TF32 bound 2e-3 (see SINGLE_PASS_TF32).  With
TE_FLAG_LINEAR_F16_SPLIT, te_set_option("gelu_split_fused", 0 / 1) must give bit-identical results.
Measured worst case per geometry on one H100 80GB HBM3 at a 400 W power limit (maps: SIMT | tensor-core sets | other):
  vit-ti       2.0e-6 | 4.5e-4 | cam_attn 2.8e-5, with BACKWARD_TF32 1.7e-3
  vit-s        1.9e-6 | 4.6e-4 | ViT_orig_LRP grad 2.9e-6 | 5.8e-4
  deit-s-dist  4.7e-6 | 5.0e-4
  vit-dh32     3.6e-6 | 3.6e-4
  vit-dh48     2.9e-6 | 3.5e-4
  vit-b-384    1.4e-5 | 4.9e-4
  bert-tiny    1.7e-6 | 1.1e-3 | rollout 7.3e-7
  bert-minilm  8.3e-7 | 2.7e-4 | attn_gradcam 4.3e-6, with BACKWARD_TF32 1.3e-3 | BERT_cls_lrp full_lrp 1.4e-7 | 4.8e-5
  bert-small   1.1e-6 | 2.4e-4 | rollout 5.5e-7 | attn_gradcam 5.1e-6, with BACKWARD_TF32 3.1e-4
Taps: probabilities <= 4.9e-6, attention gradients <= 6e-6 (fp32-grade backward) / 1.05e-3 (vit-ti, BACKWARD_TF32),
top attn_cam <= 2.7e-4, logits <= 6e-6.
"""
import collections
import functools
import re

import pytest
import torch

import bert_lrp_oracle as olrp
from oracle import bert as obert
from oracle import conditioned
from oracle import cpu as ocpu
from oracle import vit as ovit
from test_gpu_methods_tc import (FWD_TOL, GATE, NORM_TOL, VIT_C_QKV, _batched_equals_single, _bert_setup, _case_id,
                                 _gate_bert, abs_err, range_rel, rel, tol)
from transformer_explainability_b200 import _lib

pytestmark = pytest.mark.gpu

TC = _lib.FLAG_RULES_LRP_TC
BENCH = _lib.FLAG_BENCH_DEFAULT
FLAG_SETS = [0, _lib.FLAG_ALL_FAST, BENCH, BENCH | _lib.FLAG_ZPLUS_R_F16 | _lib.FLAG_BACKWARD_F16]
LRP_FLAG_SETS = FLAG_SETS + [f | TC for f in FLAG_SETS[2:]]
WORST = {}


def record(tag, what, flags, err, bound):
    print("%s %s flags %d: %.1e (bound %.0e)" % (tag, what, flags, err, bound))
    WORST[(tag, bound)] = max(WORST.get((tag, bound), 0.0), err)
    assert err < bound, "%s %s flags %d: %g >= %g" % (tag, what, flags, err, bound)


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for (tag, bound), err in sorted(WORST.items()):
        print("worst %s, bound %.0e: %.1e" % (tag, bound, err))


# With TE_FLAG_BACKWARD_TF32 the attention-gradient contractions (dctx V^T, ...) are single-pass TF32, whose stated bound is
# 2e-3 of the tensor maximum (test_gpu_tc.py::test_tc_persistent_pair_kernels).  At ViT-B width the engine's attention
# gradients stay below 1e-3 (test_gpu_engine_shapes.py); at vit-ti (3 heads) they reach 1.05e-3 and the cam_attn built from
# them 1.7e-3 absolute, against 3.0e-6 / 2.3e-5 with the same flags minus BACKWARD_TF32 (and identical with BACKWARD_F16
# added: the Linears are not the source).  So these two are held to the single-pass TF32 bound under that flag.
SINGLE_PASS_TF32 = 2e-3


def grad_tol(flags):
    return SINGLE_PASS_TF32 if flags & _lib.FLAG_BACKWARD_TF32 else 1e-4


def cam_tol(flags):
    return SINGLE_PASS_TF32 if flags & _lib.FLAG_BACKWARD_TF32 else NORM_TOL


# ---- kernel census ---------------------------------------------------------------------------------------------------------
def family(name):
    """'wg_kernel<LinProb<2, 2> >' -> 'LinProb<2, 2>'; other kernels keep their base name (tools/profile_step_kernels.py)"""
    n = name.replace("(anonymous namespace)::", "")
    m = re.search(r"wg_kernel<(\w+<[^>]*>)", n)
    if m:
        return m.group(1)
    return re.sub(r"\(.*$", "", n).replace("void ", "").strip()


def census(run):
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        run()
        torch.cuda.synchronize()
    fams = collections.Counter(family(ev.name) for ev in prof.events()
                               if ev.device_type == torch.autograd.DeviceType.CUDA)
    assert fams, "the profiler reported no CUDA kernel"
    return fams


def lin_forms(fams):
    """the FORM arguments of the LinProb<EPI, FORM> problems that ran (2 = the fp16-split forward)"""
    return {int(m.group(1)) for f in fams for m in [re.match(r"LinProb<[^,>]*,\s*(\d+)", f)] if m}


def check_census(tag, fams, present=(), absent=(), f16_forward=None):
    print("%s census: %s" % (tag, ", ".join("%s x%d" % kv for kv in sorted(fams.items()))))
    for p in present:
        assert any(f.startswith(p) for f in fams), "%s: no %s kernel ran" % (tag, p)
    for a in absent:
        assert not any(f.startswith(a) for f in fams), "%s: a %s kernel ran" % (tag, a)
    if f16_forward is not None:
        assert (2 in lin_forms(fams)) == f16_forward, "%s: fp16-split forward %s expected" % (tag, f16_forward)


# ---- ViT -------------------------------------------------------------------------------------------------------------------
VIT = {
    "vit-ti": dict(dim=192, heads=3, mlp=768),
    "vit-s": dict(dim=384, heads=6, mlp=1536),
    "deit-s-dist": dict(dim=384, heads=6, mlp=1536, distilled=True),
    "vit-dh32": dict(dim=384, heads=12, mlp=1536),
    "vit-dh48": dict(dim=384, heads=8, mlp=1536),
    "vit-b-384": dict(dim=768, heads=12, mlp=3072, img=384),
}
VIT_CASES = [("transformer_attribution", dict(start_layer=0)), ("transformer_attribution", dict(start_layer=1)),
             ("full", {}), ("rollout", dict(start_layer=0)), ("last_layer", {})]
VIT_CENSUS = {
    "vit-ti": dict(present=("LinProb", "rollout_row_kernel"), absent=("ZsProb", "ZrProb"), f16_forward=False),
    "vit-s": dict(present=("ZsProb", "ZrProb", "LinProb"), f16_forward=True),
    "deit-s-dist": dict(present=("ZsProb", "ZrProb", "LinProb"), f16_forward=True),
    "vit-dh32": dict(present=("NnProb",), absent=("NkProb",)),
    "vit-dh48": dict(absent=("NnProb", "NkProb")),
    "vit-b-384": dict(present=("aggregate_layers_vec_kernel", "extract_row_kernel"), absent=("rollout_row_kernel",)),
}
VIT_BATCHED = {"vit-ti": ("last_layer", {}), "vit-s": ("full", {}), "deit-s-dist": ("rollout", dict(start_layer=0)),
               "vit-dh32": ("transformer_attribution", dict(start_layer=1)), "vit-dh48": ("full", {}),
               "vit-b-384": ("transformer_attribution", dict(start_layer=0))}


@functools.lru_cache(maxsize=None)
def vit_setup(tag, variant="ours"):
    geom = dict(VIT[tag])
    img = geom.pop("img", 224)
    params, heads = ovit.init_params("vit_base_patch16_224", seed=5, rand_affine=True, depth=3, classes=100, img=img, **geom)
    params = conditioned.condition_vit(params, c_qkv=VIT_C_QKV)
    x = torch.randn(2, 3, img, img, generator=torch.Generator().manual_seed(6))
    ocpu.set_torch_threads()
    p64 = {k: v.double() for k, v in params.items()}
    cases = VIT_CASES if variant == "ours" else [("grad", {})]
    refs = {}
    for method, kw in cases:
        ref, idx = ovit.explain_method(p64, x.double(), heads, method, variant=variant, **kw)
        ref32, _ = ovit.explain_method(params, x, heads, method, variant=variant, **kw)
        refs[_case_id(method, kw)] = (ref, idx, rel(ref32, ref))
    taps = ovit.explain(p64, x.double(), heads, return_taps=True, variant=variant)[2] if variant == "ours" else None
    return dict(params=params, heads=heads, x=x, img=img, refs=refs, cases=cases, taps=taps, dim=geom["dim"],
                mlp=geom["mlp"], distilled=geom.get("distilled", False))


def vit_model(setup, module="ViT_LRP", **kw):
    import importlib
    mod = importlib.import_module("transformer_explainability_b200.baselines.ViT." + module)
    m = mod.VisionTransformer(img_size=setup["img"], patch_size=16, embed_dim=setup["dim"], depth=3,
                              num_heads=setup["heads"], mlp_ratio=setup["mlp"] / setup["dim"], qkv_bias=True,
                              num_classes=100, **kw)
    m.load_state_dict(setup["params"])
    return m.cuda().eval()


def run_vit_methods(tag, setup, model, flag_sets):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    lrp = LRP(model)
    x = setup["x"].cuda()
    for key, (_, _, gate) in setup["refs"].items():
        assert gate < GATE, "regime is not conditioned for %s %s: fp32 oracle vs fp64 oracle %g" % (tag, key, gate)
    for flags in flag_sets:
        model.engine_flags = flags
        for method, kw in setup["cases"]:
            ref, ridx, _ = setup["refs"][_case_id(method, kw)]
            out = lrp.generate_LRP(x, method=method, **kw)
            torch.cuda.synchronize()
            assert out.shape == ref.shape
            assert torch.equal(model.engine().tensor("logits").argmax(-1).cpu(), ridx), "%s %s: class index" % (tag, method)
            record(tag, _case_id(method, kw), flags, rel(out, ref), tol(flags))
    return lrp


@pytest.mark.parametrize("tag", list(VIT))
def test_vit_geometry(tag):
    setup = vit_setup(tag)
    model = vit_model(setup, distilled=setup["distilled"])
    lrp = run_vit_methods(tag, setup, model, FLAG_SETS)
    # per-layer taps of transformer_attribution (start_layer 0)
    x, taps, eng = setup["x"].cuda(), setup["taps"], model.engine()
    for flags in FLAG_SETS:
        _, idx, logits = eng.explain(x, flags=flags, return_logits=True)
        torch.cuda.synchronize()
        assert torch.equal(idx.cpu().long(), setup["refs"][_case_id(*VIT_CASES[0])][1])
        el = rel(logits, taps["logits"])
        ea = max(rel(model.blocks[l].attn.get_attn(), taps["cache"]["blocks"][l]["attn"]) for l in range(3))
        eg = max(rel(model.blocks[l].attn.get_attn_gradients(), taps["grads"][l]) for l in range(3))
        ec = rel(model.blocks[2].attn.get_attn_cam(), taps["cams"][2])
        print("%s taps flags %d: logits %.1e | attn %.1e | attn_grad %.1e | top attn_cam %.1e" % (tag, flags, el, ea, eg, ec))
        assert el < 1e-4 and ea < 1e-5 and eg < grad_tol(flags) and ec < 5e-2
    # a batch is a set of independent explanations
    model.engine_flags = BENCH
    method, kw = VIT_BATCHED[tag]
    out = lrp.generate_LRP(x, method=method, **kw)
    for s in range(x.shape[0]):
        _batched_equals_single(out, lrp.generate_LRP(x[s:s + 1], method=method, **kw), s)
    # the kernel mix this geometry claims
    check_census(tag, census(lambda: eng.explain(x, flags=BENCH)), **VIT_CENSUS[tag])


def test_vit_ti_baseline_cam_attn():
    """Baselines.generate_cam_attn at H = 3 (head_region_mean, head_reduce) on the hook-free ViT_new model"""
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import Baselines
    setup = vit_setup("vit-ti")
    p64 = {k: v.double() for k, v in setup["params"].items()}
    x = setup["x"]
    refs = {}
    for index in (None, 7):
        ref, ridx = ovit.baseline_cam_attn(p64, x.double(), setup["heads"], index=index)
        gate = abs_err(ovit.baseline_cam_attn(setup["params"], x, setup["heads"], index=index)[0], ref)
        assert gate < GATE, "regime is not conditioned for the vit-ti cam_attn: %g" % gate
        refs[index] = (ref, ridx)
    model = vit_model(setup, module="ViT_new", norm_layer=functools.partial(torch.nn.LayerNorm, eps=1e-6))
    base = Baselines(model)
    for flags in FLAG_SETS:
        model.engine_flags = flags
        for index, (ref, ridx) in refs.items():
            out = base.generate_cam_attn(x.cuda(), index=index)
            torch.cuda.synchronize()
            if index is None:
                assert torch.equal(model.engine().tensor("logits").argmax(-1).cpu(), ridx)
            assert out.shape == ref.shape
            assert torch.equal(torch.isnan(out.cpu()), torch.isnan(ref)), "NaN pattern of cam_attn differs"
            record("vit-ti", "cam_attn.index=%s" % index, flags, abs_err(out, ref), cam_tol(flags))


def test_vit_s_orig_lrp_grad():
    """ViT_orig_LRP (layers_lrp rules) at D = 384, with and without the tensor-core layers_lrp rule"""
    setup = vit_setup("vit-s", variant="lrp")
    model = vit_model(setup, module="ViT_orig_LRP")
    run_vit_methods("vit-s-orig-lrp", setup, model, LRP_FLAG_SETS)


# ---- BERT ------------------------------------------------------------------------------------------------------------------
BERT = {"bert-tiny": dict(dim=128, heads=2, inter=512),
        "bert-minilm": dict(dim=384, heads=12, inter=1536),
        "bert-small": dict(dim=512, heads=8, inter=2048)}
# q / k / v bias offset: the default 3 leaves the fp32 oracle's attention probabilities 1.4e-5 ... 2.8e-5 off fp64 at these
# widths, above the 1e-5 tap bound; 1 leaves them at <= 3.4e-6 and every map's regime gate at <= 4.2e-6
BERT_C_QKV = 1.0
BERT_CASES = [("LRP", dict(start_layer=0)), ("full_lrp", {}), ("attn_gradcam", {}), ("rollout", dict(start_layer=0))]
BERT_CENSUS = {"bert-tiny": dict(present=("LinProb", "ZsProb", "ZrProb", "NnProb")),
               "bert-minilm": dict(present=("LinProb", "ZsProb", "ZrProb", "NnProb")),
               "bert-small": dict(present=("ZsProb", "ZrProb", "LinProb"))}
BERT_BATCHED = {"bert-tiny": ("full_lrp", {}), "bert-minilm": ("LRP", dict(start_layer=0)), "bert-small": ("attn_gradcam", {})}


@functools.lru_cache(maxsize=None)
def bert_setup(tag):
    setup = _bert_setup(seed=51, cases=BERT_CASES, c_qkv=BERT_C_QKV, **BERT[tag])
    p64 = {k: v.double() for k, v in setup["params"].items()}
    setup["taps"] = obert.explain(p64, setup["ids"], setup["mask"], setup["heads"], start_layer=0, return_taps=True)[2]
    return setup


def bert_model(setup):
    from test_gpu_bert import make_model
    return make_model(setup["params"], setup["heads"], **setup["cfg"])


@pytest.mark.parametrize("tag", list(BERT))
def test_bert_geometry(tag):
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    setup = bert_setup(tag)
    model = bert_model(setup)
    gen = Generator(model)
    ids, mask, pad = setup["ids"].cuda(), setup["mask"].cuda(), setup["pad"]
    live = setup["mask"].bool()
    _gate_bert(setup, live)
    for flags in FLAG_SETS:
        model.engine_flags = flags
        for which, kw in BERT_CASES:
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
                record(tag, _case_id(which, kw), flags, abs_err(out, ref), cam_tol(flags))
                continue
            record(tag, _case_id(which, kw), flags, rel(out, ref), FWD_TOL if which == "rollout" else tol(flags))
            print("    %s of the range over the real tokens: %.1e" % (
                _case_id(which, kw), max(range_rel(out[s], ref[s], live[s]) for s in range(ref.shape[0]))))
    # per-layer taps of generate_LRP (start_layer 0)
    taps, eng = setup["taps"], model.engine()
    layers = model.bert.encoder.layer
    for flags in FLAG_SETS:
        maps, idx, logits = eng.explain(ids, mask, start_layer=0, flags=flags, return_logits=True)
        torch.cuda.synchronize()
        assert torch.equal(idx.cpu().long(), setup["refs"][_case_id(*BERT_CASES[0])][1])
        el = rel(logits, taps["logits"])
        ea = max(rel(layers[l].attention.self.get_attn(), taps["cache"]["layers"][l]["probs"]) for l in range(3))
        eg = max(rel(layers[l].attention.self.get_attn_gradients(), taps["grads"][l]) for l in range(3))
        ec = rel(layers[2].attention.self.get_attn_cam(), taps["cams"][2])
        print("%s taps flags %d: logits %.1e | attn %.1e | attn_grad %.1e | top attn_cam %.1e" % (tag, flags, el, ea, eg, ec))
        assert el < 1e-4 and ea < 1e-5 and eg < grad_tol(flags) and ec < 5e-2
        assert (maps[1, pad:] == 0).all(), "padded positions must get exactly zero relevance"
    model.engine_flags = BENCH
    which, kw = BERT_BATCHED[tag]
    out = getattr(gen, "generate_" + which)(ids, mask, **kw)
    for s in range(ids.shape[0]):
        _batched_equals_single(out, getattr(gen, "generate_" + which)(ids[s:s + 1], mask[s:s + 1], **kw), s)
    check_census(tag, census(lambda: eng.explain(ids, mask, start_layer=0, flags=BENCH)), **BERT_CENSUS[tag])


def test_bert_minilm_cls_lrp_full_lrp():
    """BERT_cls_lrp (layers_lrp rules) generate_full_lrp at dh 32, with and without the tensor-core layers_lrp rule"""
    from test_gpu_bert_lrp import make_model
    from transformer_explainability_b200.BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    setup = bert_setup("bert-minilm")
    p64 = {k: v.double() for k, v in setup["params"].items()}
    ids, mask, heads, pad = setup["ids"], setup["mask"], setup["heads"], setup["pad"]
    ref = olrp.generate(p64, ids, mask, heads, "full_lrp")
    gate = rel(olrp.generate(setup["params"], ids, mask, heads, "full_lrp"), ref)
    assert gate < GATE, "regime is not conditioned for bert-minilm cls_lrp full_lrp: %g" % gate
    model = make_model(setup["params"], heads, **setup["cfg"])
    gen = Generator(model)
    for flags in LRP_FLAG_SETS:
        model.engine_flags = flags
        out = gen.generate_full_lrp(ids.cuda(), mask.cuda())
        torch.cuda.synchronize()
        assert out.shape == ref.shape and not torch.isnan(out).any()
        assert float(out[1, pad:].abs().max()) == 0.0, "padded tokens must get exactly zero"
        record("bert-minilm-cls-lrp", "full_lrp", flags, rel(out, ref), 5e-3 if flags & (_lib.FLAG_TENSOR_CORES | TC) else 2e-4)


# ---- gelu_split_fused selects between two equal paths ---------------------------------------------------------------------
def _gelu_split_ab(run):
    lib = _lib.load()
    try:
        outs = []
        for on in (1, 0):
            _lib.check(lib.te_set_option(b"gelu_split_fused", on), "te_set_option")
            outs.append(run())
    finally:
        _lib.check(lib.te_set_option(b"gelu_split_fused", 1), "te_set_option")
    for a, b in zip(*outs):
        assert torch.equal(a, b), "gelu_split_fused 0 and 1 differ"


def test_gelu_split_fused_is_exact_vit_s():
    setup = vit_setup("vit-s")
    model = vit_model(setup)
    eng, x = model.engine(), setup["x"].cuda()

    def run():
        maps, _, logits = eng.explain(x, flags=BENCH, return_logits=True)
        return maps.clone(), logits.clone(), model.blocks[2].attn.get_attn_cam().clone()
    check_census("vit-s", census(run), f16_forward=True)      # the option only acts on the fp16-split forward
    _gelu_split_ab(run)


def test_gelu_split_fused_is_exact_bert_small():
    setup = bert_setup("bert-small")
    model = bert_model(setup)
    eng, ids, mask = model.engine(), setup["ids"].cuda(), setup["mask"].cuda()

    def run():
        maps, _, logits = eng.explain(ids, mask, start_layer=0, flags=BENCH, return_logits=True)
        return maps.clone(), logits.clone(), model.bert.encoder.layer[2].attention.self.get_attn_cam().clone()
    check_census("bert-small", census(run), f16_forward=True)
    _gelu_split_ab(run)
