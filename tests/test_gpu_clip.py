"""GPU: CLIP-architecture image towers on the ViT engine — pre-norm (``norm_pre``), QuickGELU, 14-pixel patches and the
image-text similarity seed of the gradient-weighted attention rollout.

- The QuickGELU epilogues on every Linear family against fp64 at the towers' widths (K = 768 / 1024, rows = batch x 50 /
  257): forward BIAS_QUICK_GELU on fp32 SIMT, 3xTF32 and the fp16 split; backward QUICK_GELU_BWD on SIMT, 3xTF32,
  single-pass TF32 and single-pass fp16.  Bounds: the Linear bounds of test_gpu_tc.py per element, QuickGELU' (|q'| <= 1.1)
  to 3e-7 absolute.  The fused fp16 split of quick_gelu(y) the fc1 epilogue emits for fc2 gives the same logits, bit for
  bit, as the stand-alone pre-pass (``gelu_split_fused`` 0).
- Random CLIP towers (``oracle.clip.init_params``: norm_pre, no patch / head bias, QuickGELU, LayerNorm eps 1e-5) at the
  geometries of ViT-B/32 (N = 50), ViT-B/16 (N = 197) and ViT-L/14 (N = 257, batch 2), 4 blocks each, stage by stage
  against the fp64 oracle on the engine's own samples: the tokens after norm_pre, the attention probabilities, d s / d A
  and the maps, plus the similarity, under flag sets 0, FLAG_ALL_FAST and FLAG_BENCH_DEFAULT.  Bounds relative to the
  tensor maximum: forward 1e-5 (tensor cores 1e-4), gradients and maps 2e-4 SIMT / 5e-3 tensor cores, as
  test_gpu_attn_grad_rollout.py; the similarity 1e-6 of logit_scale (1e-5 on the tensor cores).
- The pre-norm / QuickGELU classifier facade (``ViT_LRP.VisionTransformer(pre_norm=True, act_layer="quick_gelu")``),
  conditioned as test_gpu_methods_tc.py conditions (norm_pre's bias carries the token offset): transformer_attribution,
  full (pixels; patch 16 and 14), alpha = 0.5 and attn_grad_rollout against the fp64 oracle (``oracle.clip.architecture``
  around oracle.vit / oracle.alphabeta / oracle.attn_grad_rollout), with the regime gate of those tests.
- TE_FLAG_SIMILARITY_SEED without TE_FLAG_ATTN_GRAD_ROLLOUT, and in te_vit_explain, is refused; batched equals per-sample
  and chunked; a poisoned workspace gives bit-identical similarities and maps.
- The fixture's tiny towers (tests/golden/clip.npz: transformers' similarity and d s / d A, the rule's maps) under every
  flag set; ``CLIPExplainer`` on a saved Hugging Face directory against the model's own logits_per_image; the
  ``clip_visualization`` command end to end against ``CLIPExplainer`` on the command's preprocessing.
"""
import pytest
import torch

from oracle import alphabeta as oab
from oracle import attn_grad_rollout as agr
from oracle import clip as oclip
from oracle import conditioned
from oracle import cpu as ocpu
from oracle import vit as ovit
from transformer_explainability_b200 import _lib, ops
from transformer_explainability_b200.engine import ViTEngine, vit_config

pytestmark = pytest.mark.gpu

AGR = _lib.FLAG_ATTN_GRAD_ROLLOUT
FLAG_SETS = [0, _lib.FLAG_ALL_FAST, _lib.FLAG_BENCH_DEFAULT]
GATE = 1e-4
LIN_BOUND = {"simt": lambda K: 3e-6, "3xtf32": lambda K: 1.5e-8 * K + 2e-6, "f16_split": lambda K: 1.5e-8 * K + 2e-6,
             "tf32": lambda K: 2e-3, "f16": lambda K: 2e-3}
QGELU_GRAD = 3e-7


def tol(flags):
    return 5e-3 if flags & _lib.FLAG_TENSOR_CORES else 2e-4


def fwd_tol(flags):
    return 1e-4 if flags & _lib.FLAG_TENSOR_CORES else 1e-5


def rel(a, b):
    b = torch.as_tensor(b).double().cpu()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def _qgelu64(y):
    return y * torch.sigmoid(1.702 * y)


def _qgelu_grad64(x):
    s = torch.sigmoid(1.702 * x)
    return s * (1 + 1.702 * x * (1 - s))


# ---- the QuickGELU epilogues ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [768, 1024])
@pytest.mark.parametrize("rows", [100, 514])
def test_quick_gelu_forward_epilogue(rows, K):
    N = 256
    g = torch.Generator(device="cuda").manual_seed(rows + K)
    x = torch.randn(rows, K, generator=g, device="cuda") * torch.logspace(-2, 2, rows, device="cuda")[:, None]
    w = torch.randn(N, K, generator=g, device="cuda") * 0.05
    b = torch.randn(N, generator=g, device="cuda") * 0.1
    y64 = x.double() @ w.double().T + b.double()
    scale = x.double().abs() @ w.double().abs().T + b.double().abs()
    for family in ("simt", "3xtf32", "f16_split"):
        bound = LIN_BOUND[family](K)
        y, y2 = ops.linear_forward_epi(x, w, b, epi="bias_quick_gelu", family=family)
        y_ref, _ = ops.linear_forward_epi(x, w, b, epi="bias", family=family)
        torch.cuda.synchronize()
        ey = ((y.double() - y64).abs() / scale).max().item()
        e2 = ((y2.double() - _qgelu64(y64)).abs() / (1.1 * scale)).max().item()
        print("QuickGELU fwd %s rows %d K %d: y %.2e y2 %.2e (bound %.1e)" % (family, rows, K, ey, e2, bound))
        assert torch.equal(y, y_ref), family                        # y is the BIAS epilogue's, bit for bit
        assert ey < bound and e2 < bound + 5e-7, family


@pytest.mark.parametrize("K", [768, 1024])
@pytest.mark.parametrize("rows", [100, 514])
def test_quick_gelu_backward_epilogue(rows, K):
    N = 256
    g = torch.Generator(device="cuda").manual_seed(rows * 7 + K)
    dy = torch.randn(rows, K, generator=g, device="cuda")
    w = torch.randn(K, N, generator=g, device="cuda") * 0.05
    e0 = torch.rand(rows, N, generator=g, device="cuda") * 40 - 20
    e0.view(-1)[:8] = torch.tensor([0.0, 1e-6, -1e-6, 1.5, -1.5, 60.0, -60.0, -100.0], device="cuda")
    gp = _qgelu_grad64(e0.double())
    v64 = dy.double() @ w.double()
    scale = dy.double().abs() @ w.double().abs()
    for family in ("simt", "3xtf32", "tf32", "f16"):
        bound = LIN_BOUND[family](K)
        dx = ops.linear_backward_epi(dy, w, e0, epi="quick_gelu_bwd", family=family)
        v = ops.linear_backward_epi(dy, w, None, epi="store", family=family)
        torch.cuda.synchronize()
        e_full = ((dx.double() - v64 * gp).abs() / (scale * ((bound + 1.2e-7) * gp.abs() + QGELU_GRAD))).max().item()
        live = v != 0
        grad_err = (dx.double()[live] / v.double()[live] - gp[live]).abs().max().item()
        print("QuickGELU bwd %s rows %d K %d: %.2f of the bound, QuickGELU' abs err %.2e" % (family, rows, K, e_full, grad_err))
        assert torch.isfinite(dx).all(), family
        assert e_full < 1 and grad_err < QGELU_GRAD + 1.2e-7, family


# ---- random CLIP towers, stage by stage -------------------------------------------------------------------------------
TOWERS = {"B32": dict(patch=32, dim=768, heads=12, mlp=3072, embed=512, batch=3),
          "B16": dict(patch=16, dim=768, heads=12, mlp=3072, embed=512, batch=2),
          "L14": dict(patch=14, dim=1024, heads=16, mlp=4096, embed=768, batch=2)}
DEPTH = 4
LOGIT_SCALE = 100.0


def _tower_cfg(c, depth=DEPTH, act="quick_gelu"):
    return vit_config(224, c["patch"], 3, c["embed"], c["dim"], depth, c["heads"], c["mlp"] / c["dim"], eps_block=1e-5,
                      eps_final=1e-5, pre_norm=True, act=act)


@pytest.fixture(scope="module", params=sorted(TOWERS))
def tower(request):
    c = TOWERS[request.param]
    params, heads = oclip.init_params(patch=c["patch"], dim=c["dim"], depth=DEPTH, heads=c["heads"], mlp=c["mlp"],
                                      embed=c["embed"], seed=3)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(c["batch"], 3, 224, 224, generator=g)
    text = torch.randn(c["batch"], c["embed"], generator=g)
    eng = ViTEngine(_tower_cfg(c), params)
    return dict(name=request.param, c=c, params=params, heads=heads, x=x, text=text, eng=eng)


def _engine_run(eng, x, text, flags, start_layer=0):
    eng.forward(x.cuda(), flags=flags)
    sim = eng.similarity(text.cuda(), LOGIT_SCALE)
    maps, idx = eng.attribute(start_layer=start_layer, flags=flags, similarity_seeded=True)
    torch.cuda.synchronize()
    return sim, maps, idx


@pytest.mark.parametrize("flags", FLAG_SETS)
def test_tower_stages_against_fp64(tower, flags):
    """Each stage of the engine against fp64 evaluated on the engine's own input to that stage: norm_pre's output from the
    images; block l's probabilities from the engine's block input (the oracle's own forward from there); d s / d A and the
    maps of the whole fp64 chain (the gradients flow through every block above)."""
    eng, p, heads, x, text = tower["eng"], tower["params"], tower["heads"], tower["x"], tower["text"]
    sim, maps, idx = _engine_run(eng, x, text, flags)
    p64 = {k: v.double() for k, v in p.items()}
    ocpu.set_torch_threads()
    attns, grads, s64, cache = oclip.similarity_taps(p64, x.double(), heads, text.double(), LOGIT_SCALE)
    e_pre = rel(eng.tensor("x_in", 0), cache["x_pre"])
    assert e_pre < fwd_tol(flags), e_pre
    cfg = cache["cfg"]
    for l in range(DEPTH):
        x_l = eng.tensor("x_in", l).double().cpu()
        _, c = oclip.block_forward(p64, cfg, l, x_l, "quick_gelu")
        e_p = rel(eng.tensor("attn", l), c["attn"])
        e_g = rel(eng.tensor("attn_grad", l), grads[l])
        print("%s flags %d block %d: probs %.1e, ds/dA %.1e" % (tower["name"], flags, l, e_p, e_g))
        assert e_p < fwd_tol(flags) and e_g < tol(flags), (l, e_p, e_g)
    ref = agr.vit_map(attns, grads, 0, prefix=1)
    # the similarity's error in units of logit_scale: the error of the cosine (a similarity near 0 has no relative scale)
    e_m, e_s = rel(maps, ref), ((sim.double().cpu() - s64).abs() / LOGIT_SCALE).max().item()
    print("%s flags %d: maps %.1e, similarity %.1e of logit_scale" % (tower["name"], flags, e_m, e_s))
    assert e_m < tol(flags) and e_s < 1e-6 * (10 if flags & _lib.FLAG_TENSOR_CORES else 1)
    assert torch.equal(idx.cpu(), torch.full_like(idx.cpu(), -1))          # index is neither read nor written


def _seeded_in_chunks(eng, x, text, flags, sizes):
    """the batch explained chunk by chunk (each chunk its own forward, seed and attribute), concatenated"""
    sims, maps, s = [], [], 0
    for n in sizes:
        si, mi, _ = _engine_run(eng, x[s:s + n], text[s:s + n], flags)
        sims.append(si.clone())
        maps.append(mi.clone())
        s += n
    return torch.cat(sims), torch.cat(maps)


def test_tower_batched_equals_per_sample_chunked_and_poisoned(tower, monkeypatch):
    """Batched equals per-sample and chunked (the batch split 2 + rest, and one by one); with every workspace and output
    the engine allocates replaced by test_gpu_poison.py's poisoned allocations (0xFF and 0x5A, 2 MiB guards), the
    similarities and maps are bit-identical to a normal run and every guard still holds its pattern."""
    import os
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    from test_gpu_poison import PoisonTorch
    from transformer_explainability_b200 import engine as engine_mod
    eng, x, text = tower["eng"], tower["x"], tower["text"]
    flags = _lib.FLAG_BENCH_DEFAULT
    sim, maps, _ = _engine_run(eng, x, text, flags)
    sim, maps = sim.clone(), maps.clone()
    B = x.shape[0]
    for sizes in ([1] * B, [2, B - 2] if B > 2 else [1, B - 1]):
        s_c, m_c = _seeded_in_chunks(eng, x, text, flags, sizes)
        assert rel(m_c, maps) < 1e-6 and rel(s_c, sim) < 1e-6, sizes
    for pattern in (0xFF, 0x5A):
        proxy = PoisonTorch(pattern)
        with monkeypatch.context() as mp:
            mp.setattr(engine_mod, "torch", proxy)
            eng._ws = None                                   # a fresh, poisoned workspace
            eng.forward(x.cuda(), flags=flags)
            sim_p = eng.similarity(text.cuda(), LOGIT_SCALE)
            maps_p, _ = eng.attribute(flags=flags, similarity_seeded=True)
            torch.cuda.synchronize()
        assert torch.equal(sim_p.view(torch.int32), sim.view(torch.int32)), pattern
        assert torch.equal(maps_p.view(torch.int32), maps.view(torch.int32)), pattern
        assert proxy.broken_guards() == 0, pattern
    eng._ws = None
    # start_layer > 0 and the deepest start
    for sl in (1, DEPTH - 1):
        _, m, _ = _engine_run(eng, x, text, 0, start_layer=sl)
        p64 = {k: v.double() for k, v in tower["params"].items()}
        ref, _ = oclip.explain_similarity(p64, x.double(), tower["heads"], text.double(), LOGIT_SCALE, start_layer=sl)
        assert rel(m, ref) < tol(0), sl


def test_seed_belongs_to_the_current_forward(tower):
    """A seeded attribute() after another forward, or after a class attribute() overwrote the seed, is refused; a second
    seeded call on the same seed (another start_layer) is not."""
    eng, x, text = tower["eng"], tower["x"].cuda(), tower["text"].cuda()
    eng.forward(x)
    with pytest.raises(RuntimeError):
        eng.attribute(similarity_seeded=True)
    eng.similarity(text, LOGIT_SCALE)
    eng.forward(x.flip(0))
    with pytest.raises(RuntimeError):
        eng.attribute(similarity_seeded=True)
    eng.similarity(text, LOGIT_SCALE)
    eng.attribute(similarity_seeded=True)
    eng.attribute(start_layer=1, similarity_seeded=True)
    eng.attribute(flags=AGR)                                 # class rollout: its one-hot replaces the seed
    with pytest.raises(RuntimeError):
        eng.attribute(similarity_seeded=True)
    eng.similarity(text, LOGIT_SCALE)
    eng.explain(x, flags=AGR)
    with pytest.raises(RuntimeError):
        eng.attribute(flags=_lib.FLAG_SIMILARITY_SEED | AGR)


def test_similarity_seed_flag_needs_grad_rollout(tower):
    eng = tower["eng"]
    eng.forward(tower["x"].cuda())
    eng.similarity(tower["text"].cuda(), LOGIT_SCALE)
    with pytest.raises(_lib.TeError) as e:
        eng.attribute(flags=_lib.FLAG_SIMILARITY_SEED)
    assert e.value.status == -1 and "TE_FLAG_ATTN_GRAD_ROLLOUT" in str(e.value)
    with pytest.raises(_lib.TeError):
        eng.attribute(flags=_lib.FLAG_SIMILARITY_SEED | AGR, alpha=0.5)
    with pytest.raises(_lib.TeError) as e:                  # explain() runs its own forward: no seed between
        eng.explain(tower["x"].cuda(), flags=_lib.FLAG_SIMILARITY_SEED | AGR)
    assert e.value.status == -1


def test_fused_quick_gelu_split_matches_prepass(tower):
    eng, x = tower["eng"], tower["x"].cuda()
    fused = eng.forward(x, flags=_lib.FLAG_BENCH_DEFAULT).clone()
    lib = _lib.load()
    assert lib.te_set_option(b"gelu_split_fused", 0) == 0
    try:
        prepass = eng.forward(x, flags=_lib.FLAG_BENCH_DEFAULT).clone()
    finally:
        lib.te_set_option(b"gelu_split_fused", 1)
    assert torch.equal(fused, prepass)


# ---- the pre-norm / QuickGELU classifier facade ---------------------------------------------------------------------------
def _facade_setup(patch, dim, heads, mlp, act):
    params, _ = ovit.init_params("vit_base_patch16_224", seed=21, rand_affine=True, depth=3, classes=100, patch=patch, dim=dim,
                                 heads=heads, mlp=mlp)
    params = conditioned.condition_vit(params, c_qkv=1.0)
    g = torch.Generator().manual_seed(22)
    params["norm_pre.weight"] = 1 + 0.2 * torch.randn(dim, generator=g)
    params["norm_pre.bias"] = 4.0 + 0.05 * torch.randn(dim, generator=g)   # the token offset of condition_vit, after norm_pre
    from transformer_explainability_b200.baselines.ViT.ViT_LRP import VisionTransformer
    m = VisionTransformer(img_size=224, patch_size=patch, embed_dim=dim, depth=3, num_heads=heads, mlp_ratio=mlp / dim,
                          qkv_bias=True, num_classes=100, pre_norm=True, act_layer=act)
    m.load_state_dict(params)
    x = torch.randn(2, 3, 224, 224, generator=g)
    return m.cuda().eval(), params, x


FACADE_CASES = [("transformer_attribution", 1.0), ("full", 1.0), ("transformer_attribution", 0.5), ("attn_grad_rollout", 1.0)]


@pytest.mark.parametrize("act", ["quick_gelu", "gelu"])
@pytest.mark.parametrize("patch,dim,heads,mlp", [(16, 768, 12, 3072), (14, 1024, 16, 4096)])
def test_prenorm_classifier_facade(patch, dim, heads, mlp, act):
    from transformer_explainability_b200.baselines.ViT.ViT_explanation_generator import LRP
    m, params, x = _facade_setup(patch, dim, heads, mlp, act)
    p64 = {k: v.double() for k, v in params.items()}
    ocpu.set_torch_threads()
    refs = {}
    with oclip.architecture(act):
        for method, alpha in FACADE_CASES:
            if method == "attn_grad_rollout":
                ref, idx = agr.explain_vit(p64, x.double(), heads)
                ref32, _ = agr.explain_vit(params, x, heads)
            else:
                ref, idx = oab.vit_explain_method(p64, x.double(), heads, method, alpha)
                ref32, _ = oab.vit_explain_method(params, x, heads, method, alpha)
            gate = rel(ref32, ref)
            assert gate < GATE, "regime is not conditioned for %s: fp32 oracle vs fp64 oracle %g" % (method, gate)
            refs[(method, alpha)] = (ref, idx)
    for flags in FLAG_SETS:
        m.engine_flags = flags
        for (method, alpha), (ref, idx) in refs.items():
            if method == "attn_grad_rollout":
                out = LRP(m).generate_attn_grad_rollout(x.cuda())
            else:
                logits = m(x.cuda())
                assert torch.equal(logits.argmax(-1).cpu(), idx)
                seed = torch.nn.functional.one_hot(idx, 100).float().cuda()
                out = m.relprop(seed, method=method, alpha=alpha)
            torch.cuda.synchronize()
            e = rel(out, ref)
            print("facade patch %d %s flags %d %s alpha %g: %.1e (bound %.0e)" % (patch, act, flags, method, alpha, e, tol(flags)))
            assert out.shape == ref.shape and e < tol(flags), (flags, method, alpha, e)


# ---- a local Hugging Face CLIP directory, end to end ------------------------------------------------------------------------
@pytest.mark.parametrize("act,patch", [("quick_gelu", 14), ("gelu", 16)])
def test_clip_explainer_on_a_saved_directory(tmp_path, act, patch):
    """``CLIPExplainer`` on a tiny ``transformers.CLIPModel`` saved to disk: the similarities against the model's own
    ``logits_per_image`` (fp32 model, one text row per image) to fp32 rounding, the maps against the fp64 oracle of the
    same weights, and a second prompt on the same forward equal to a fresh run."""
    import sys
    sys.path.insert(0, __import__("os").path.dirname(__file__))
    from test_clip import _tiny_clip
    from transformer_explainability_b200 import clip as tclip
    m = _tiny_clip(act, patch, seed=7).float()
    m.save_pretrained(tmp_path)
    vc = m.config.vision_config
    g = torch.Generator().manual_seed(8)
    x = torch.randn(3, 3, vc.image_size, vc.image_size, generator=g)
    texts = torch.randn(2, m.config.projection_dim, generator=g)
    for flags in (0, _lib.FLAG_BENCH_DEFAULT):
        ex = tclip.CLIPExplainer(str(tmp_path), flags=flags)
        maps, sim = ex.generate_attn_grad_rollout(x.cuda(), texts[0])
        maps2, sim2 = ex.explain_forwarded(texts[1].cuda())
        again, sim_again = ex.generate_attn_grad_rollout(x.cuda(), texts[1])
        torch.cuda.synchronize()
        assert torch.equal(maps2, again) and torch.equal(sim2, sim_again)
        with torch.no_grad():
            emb = m.visual_projection(m.vision_model(pixel_values=x).pooler_output)
            lpi = ex.logit_scale * (emb / emb.norm(dim=-1, keepdim=True)) @ (texts / texts.norm(dim=-1, keepdim=True)).T
        assert torch.allclose(sim.cpu(), lpi[:, 0], rtol=2e-5, atol=2e-5 * lpi.abs().max())
        assert torch.allclose(sim2.cpu(), lpi[:, 1], rtol=2e-5, atol=2e-5 * lpi.abs().max())
        sd, scale = tclip.engine_state_dict({k: v.double() for k, v in m.state_dict().items()}, vc.num_hidden_layers)
        ref, s64 = oclip.explain_similarity(sd, x.double(), vc.num_attention_heads, texts[:1].expand(3, -1).double(), scale,
                                            act=act, norm_eps=vc.layer_norm_eps)
        e = rel(maps, ref)
        print("CLIPExplainer %s patch %d flags %d: maps %.1e" % (act, patch, flags, e))
        assert maps.shape == (3, (vc.image_size // patch) ** 2) and e < tol(0)


def test_clip_visualization_command_end_to_end(tmp_path):
    """The command on a tiny saved directory: one overlay per image x prompt, ``similarities.json`` equal to
    ``CLIPExplainer`` on the command's own preprocessing and prompts, and the overlays equal to that run's."""
    import json
    import os
    import sys
    import numpy as np
    from PIL import Image
    sys.path.insert(0, os.path.dirname(__file__))
    from test_clip import save_tiny_clip_dir
    from transformer_explainability_b200 import clip as tclip, clip_visualization as cv, hdf5_writer
    from transformer_explainability_b200.visualization import relevance_to_heatmap, render_overlays
    model_dir, imgs, out = tmp_path / "clip", tmp_path / "imgs", tmp_path / "out"
    save_tiny_clip_dir(model_dir)
    imgs.mkdir()
    rng = np.random.default_rng(0)
    for name, (h, w) in (("wide", (61, 97)), ("tall", (90, 57)), ("square", (56, 56))):
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(imgs / (name + ".png"))
    prompts = ["a dog", "a photo of a cat"]
    written = cv.main(["--model-dir", str(model_dir), "--images", str(imgs), "--text"] + prompts +
                      ["--output-dir", str(out), "--batch-size", "2"])
    assert len(written) == 6 and all(os.path.exists(p) for p in written)
    res = json.load(open(out / "similarities.json"))
    assert res["prompts"] == prompts
    ex = tclip.CLIPExplainer(str(model_dir))
    text = ex.encode_text(prompts).cuda()
    paths = sorted(str(imgs / f) for f in os.listdir(imgs))
    packed, sizes, offsets, _ = hdf5_writer.pack_images([(hdf5_writer.read_rgb(p), 0) for p in paths])
    x = cv.prepare_batch(packed.cuda(), sizes.numpy(), offsets.numpy(), 56)
    ex.engine.forward(x)
    for j in range(len(prompts)):
        maps, sim = ex.explain_forwarded(text[j])
        over = render_overlays(x, relevance_to_heatmap(maps, grid=4, scale=14)).cpu().numpy()
        for i, p in enumerate(paths):
            stem = os.path.splitext(os.path.basename(p))[0]
            assert res[stem]["similarities"][j] == pytest.approx(float(sim[i]), rel=1e-6, abs=1e-6)
            assert np.array_equal(np.asarray(Image.open(out / ("%s_%d.png" % (stem, j)))), over[i])


@pytest.mark.parametrize("flags", FLAG_SETS + [_lib.FLAG_BENCH_DEFAULT | _lib.FLAG_BACKWARD_F16])
@pytest.mark.parametrize("key", ["q", "g", "t"])
def test_tiny_clip_against_fixture(key, flags):
    """The engine on the fixture's tiny towers (tests/golden/clip.npz: transformers' similarity and d s / d A, the rule's
    maps) at start_layer 0 and 1.  At width 32 (q, g) every flag set runs the SIMT kernels; tower t (width 128, heads of 64,
    MLP 512) takes the tensor-core Linear families (3xTF32, the fp16 split with its fused QuickGELU split, single-pass
    TF32 / fp16 backward) and the tensor-core attention contractions under the tensor-core flag sets."""
    import os
    import sys
    import numpy as np
    sys.path.insert(0, os.path.dirname(__file__))
    from test_clip import GOLDEN, golden_model
    z = np.load(GOLDEN)
    sd, heads, scale, eps, act, x, text = golden_model(z, key)
    D, img = sd["cls_token"].shape[-1], x.shape[-1]
    P = sd["patch_embed.proj.weight"].shape[-1]
    mlp = sd["blocks.0.mlp.fc1.weight"].shape[0]
    L = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
    cfg = vit_config(img, P, 3, text.shape[1], D, L, heads, mlp / D, eps_block=eps, eps_final=eps, pre_norm=True, act=act)
    eng = ViTEngine(cfg, sd)
    for sl in (0, 1):
        eng.forward(x.cuda(), flags=flags)
        sim = eng.similarity(text.cuda(), scale)
        maps, _ = eng.attribute(start_layer=sl, flags=flags, similarity_seeded=True)
        torch.cuda.synchronize()
        ref_s = torch.from_numpy(z[key + ".hf.similarity"])
        assert ((sim.double().cpu() - ref_s).abs() / scale).max() < 1e-6 * (10 if flags & _lib.FLAG_TENSOR_CORES else 1)
        for l in range(sl, L):
            assert rel(eng.tensor("attn_grad", l), z["%s.hf.grad.%d" % (key, l)]) < tol(flags), l
        e = rel(maps, z["%s.maps.sl%d" % (key, sl)])
        print("tiny CLIP %s flags %d start_layer %d: maps %.1e" % (key, flags, sl, e))
        assert e < tol(flags)


# ---- Pillow's bicubic resize (CLIP's preprocessing) ----------------------------------------------------------------------------
BICUBIC_CASES = [((375, 500), (224, 298)), ((500, 375), (298, 224)), ((61, 97), (224, 352)), ((97, 61), (352, 224)),
                 ((224, 224), (224, 224)), ((5, 3), (17, 11)), ((299, 301), (223, 225)), ((1, 1), (3, 3)),
                 ((1500, 9), (37, 5)), ((1200, 801), (335, 224)), ((3, 700), (224, 52267 // 1000))]


def test_prepare_images_bicubic_equals_pil():
    """``ops.prepare_images(resample="bicubic")`` on one ragged batch against ``PIL.Image.resize(..., BICUBIC)`` +
    ``ToTensor``, bit for bit, per output size (down- and upscaling, odd sizes, 1 x 1, an image tall enough for Pillow to
    resize vertically first); each image alone gives the bits it gets in the batch; bilinear through the same entry point
    is unchanged."""
    import numpy as np
    from PIL import Image
    from transformer_explainability_b200 import hdf5_writer
    rng = np.random.default_rng(1)
    imgs = [Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)) for (h, w), _ in BICUBIC_CASES]
    for i, (_, (oh, ow)) in enumerate(BICUBIC_CASES):
        idx = [j for j, (_, o) in enumerate(BICUBIC_CASES) if o == (oh, ow)]
        if idx[0] != i:
            continue
        packed, sizes, offsets, _ = hdf5_writer.pack_images([(imgs[j], 0) for j in idx])
        out01, norm = ops.prepare_images(packed.cuda(), sizes.numpy(), offsets.numpy(), (oh, ow), mean=(0.1, 0.2, 0.3),
                                         std=(0.5, 0.25, 0.125), resample="bicubic")
        torch.cuda.synchronize()
        for n, j in enumerate(idx):
            ref = torch.from_numpy(np.asarray(imgs[j].resize((ow, oh), Image.BICUBIC))).permute(2, 0, 1).float() / 255
            assert torch.equal(out01[n].cpu(), ref), BICUBIC_CASES[j]
            want = (ref - torch.tensor([0.1, 0.2, 0.3])[:, None, None]) / torch.tensor([0.5, 0.25, 0.125])[:, None, None]
            assert torch.equal(norm[n].cpu(), want), BICUBIC_CASES[j]
            p1, s1, o1, _ = hdf5_writer.pack_images([(imgs[j], 0)])
            alone, _ = ops.prepare_images(p1.cuda(), s1.numpy(), o1.numpy(), (oh, ow), resample="bicubic")
            assert torch.equal(alone[0], out01[n])
        bil, _ = ops.prepare_images(packed.cuda(), sizes.numpy(), offsets.numpy(), (oh, ow))
        for n, j in enumerate(idx):
            ref = torch.from_numpy(np.asarray(imgs[j].resize((ow, oh), Image.BILINEAR))).permute(2, 0, 1).float() / 255
            assert torch.equal(bil[n].cpu(), ref)


def test_clip_command_preprocessing_equals_clips():
    """The command's ``prepare_batch`` against CLIP's own preprocessing on the host: shorter side to 224 with PIL bicubic
    (torchvision's ``Resize(224)`` sizes), center crop 224 (``CenterCrop``'s offsets), ToTensor, CLIP's mean / std, in
    fp32 — bit for bit."""
    import numpy as np
    from PIL import Image
    from transformer_explainability_b200 import clip_visualization as cv, hdf5_writer
    rng = np.random.default_rng(2)
    imgs = [Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
            for h, w in ((375, 500), (500, 333), (224, 224), (100, 150), (801, 1200), (300, 301))]
    packed, sizes, offsets, _ = hdf5_writer.pack_images([(im, 0) for im in imgs])
    x = cv.prepare_batch(packed.cuda(), sizes.numpy(), offsets.numpy(), 224).cpu()
    mean, std = torch.tensor(cv.CLIP_MEAN)[:, None, None], torch.tensor(cv.CLIP_STD)[:, None, None]
    for i, im in enumerate(imgs):
        w, h = im.size
        rh, rw = (int(224 * h / w), 224) if w <= h else (224, int(224 * w / h))
        r = np.asarray(im.resize((rw, rh), Image.BICUBIC))
        top, left = int(round((rh - 224) / 2.0)), int(round((rw - 224) / 2.0))
        ref = torch.from_numpy(r[top:top + 224, left:left + 224].copy()).permute(2, 0, 1).float() / 255
        assert torch.equal(x[i], (ref - mean) / std), im.size
