"""CPU: the CLIP image-tower pieces that need no GPU.

- ``oracle.clip`` against ``transformers.CLIPModel`` itself (tiny random models in fp64 with eager attention, once with
  QuickGELU at patch 14 and once with GELU at patch 16): the similarity against ``logits_per_image``, the attention
  probabilities against ``output_attentions``, d s / d A against autograd through the model's own attention tensors, and
  the maps of the unchanged ``oracle.attn_grad_rollout`` rule on those tensors.  This also pins the key mapping of
  ``clip.engine_state_dict`` (q / k / v -> qkv, pre_layrnorm -> norm_pre, post_layernorm -> norm, visual_projection -> head).
  transformers' eager attention takes its softmax in fp32 whatever the model's dtype, so the two agree to ~1e-8, not to
  fp64 rounding: the bounds are 1e-6.
- The weight table with ``norm_pre``, a zeroed config tail giving the weight table and workspace size of the model
  without it, patch 14 accepted, an unknown activation refused (host-only library calls).
- ``clip.read_config`` / ``load_weights`` on a saved directory.
"""
import ctypes

import pytest
import torch

from oracle import attn_grad_rollout as agr
from oracle import clip as oclip
from transformer_explainability_b200 import _lib
from transformer_explainability_b200 import clip as tclip
from transformer_explainability_b200.engine import vit_config


def _tiny_clip(act, patch, seed):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.CLIPConfig(
        text_config=dict(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=2,
                         max_position_embeddings=16),
        vision_config=dict(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=4,
                           image_size=56 if patch == 14 else 64, patch_size=patch, hidden_act=act),
        projection_dim=24)
    torch.manual_seed(seed)
    m = transformers.CLIPModel._from_config(cfg, attn_implementation="eager").double().eval()
    with torch.no_grad():                       # non-trivial LayerNorm affines and biases
        for n, p in m.named_parameters():
            if "layer_norm" in n or "layrnorm" in n:
                p.add_(0.1 * torch.randn_like(p))
    return m


@pytest.mark.parametrize("act,patch", [("quick_gelu", 14), ("gelu", 16)])
def test_oracle_matches_transformers(act, patch):
    m = _tiny_clip(act, patch, seed=1 if act == "gelu" else 2)
    vc = m.config.vision_config
    B = 3
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 3, vc.image_size, vc.image_size, generator=g, dtype=torch.float64)
    text = torch.randn(B, m.config.projection_dim, generator=g, dtype=torch.float64)
    sd, scale = tclip.engine_state_dict(m.state_dict(), vc.num_hidden_layers)
    assert scale == pytest.approx(float(m.logit_scale.detach().exp()), rel=1e-12)

    with torch.enable_grad():
        out = m.vision_model(pixel_values=x, output_attentions=True)
        emb = m.visual_projection(out.pooler_output)
        s_hf = oclip.similarity(emb, text, scale)
        grads_hf = torch.autograd.grad(s_hf.sum(), out.attentions)
    attns, grads, s, cache = oclip.similarity_taps(sd, x, vc.num_attention_heads, text, scale, act=act,
                                                   norm_eps=vc.layer_norm_eps)
    # CLIP's own logits_per_image of each image with its text row
    emb_n = emb / emb.norm(dim=-1, keepdim=True)
    t_n = text / text.norm(dim=-1, keepdim=True)
    assert torch.allclose(s, (scale * emb_n @ t_n.T).diagonal(), rtol=1e-6, atol=0)
    assert torch.allclose(s, s_hf.detach(), rtol=1e-6, atol=0)
    for a, a_hf, gr, g_hf in zip(attns, out.attentions, grads, grads_hf):
        assert torch.allclose(a, a_hf.detach(), rtol=0, atol=1e-7)
        assert torch.allclose(gr, g_hf, rtol=0, atol=1e-6 * g_hf.abs().max())
    maps = agr.vit_map(attns, grads, 0, prefix=1)
    maps_hf = agr.vit_map([a.detach() for a in out.attentions], list(grads_hf), 0, prefix=1)
    assert maps.shape == (B, (vc.image_size // patch) ** 2)
    assert torch.allclose(maps, maps_hf, rtol=0, atol=1e-6 * maps_hf.abs().max())


def _table(cfg):
    lib = _lib.load()
    c = ctypes.byref(cfg)
    n = _lib.check(lib.te_vit_num_weights(c))
    return [(lib.te_vit_weight_name(c, i).decode(), lib.te_vit_weight_numel(c, i), lib.te_vit_weight_offset(c, i))
            for i in range(n)], lib.te_vit_weight_total(c)


def test_weight_table_norm_pre_and_zeroed_tail():
    lib = _lib.load()
    base = vit_config(224, 16, 3, 512, 768, 12, 12, 4.0)
    clip = vit_config(224, 16, 3, 512, 768, 12, 12, 4.0, pre_norm=True, act="quick_gelu")
    t0, n0 = _table(base)
    t1, n1 = _table(clip)
    names0, names1 = [t[0] for t in t0], [t[0] for t in t1]
    i = names1.index("pos_embed")
    assert names1[i + 1:i + 3] == ["norm_pre.weight", "norm_pre.bias"]
    assert names1[:i + 1] + names1[i + 3:] == names0
    assert [t[1] for t in t1 if t[0].startswith("norm_pre")] == [768, 768]
    assert n1 == n0 + 2 * 768
    # a config written by a caller that knows only the first eleven fields: the tail is zero
    old = _lib.TeVitConfig(*[getattr(base, f) for f, _ in _lib.TeVitConfig._fields_[:11]])
    assert old.pre_norm == 0 and old.act == 0
    assert _table(old) == (t0, n0)
    for b in (1, 7, 64):
        ws = lib.te_vit_workspace_bytes(ctypes.byref(base), b)
        assert ws > 0
        assert lib.te_vit_workspace_bytes(ctypes.byref(old), b) == ws
        assert lib.te_vit_workspace_bytes(ctypes.byref(clip), b) == ws


def test_patch_14_accepted_and_bad_tail_refused():
    lib = _lib.load()
    l14 = vit_config(224, 14, 3, 768, 1024, 24, 16, 4.0, pre_norm=True, act="quick_gelu")
    t, _ = _table(l14)
    assert dict((n, k) for n, k, _ in t)["patch_embed.proj.weight"] == 1024 * 3 * 14 * 14
    assert dict((n, k) for n, k, _ in t)["pos_embed"] == 257 * 1024
    assert lib.te_vit_workspace_bytes(ctypes.byref(l14), 2) > 0
    for field, value in (("act", 2), ("pre_norm", 2)):
        bad = vit_config(224, 14, 3, 768, 1024, 24, 16, 4.0)
        setattr(bad, field, value)
        assert lib.te_vit_num_weights(ctypes.byref(bad)) < 0
        assert lib.te_vit_workspace_bytes(ctypes.byref(bad), 1) < 0
    with pytest.raises(ValueError):
        vit_config(act="relu")


def test_read_config_and_weights_of_a_saved_directory(tmp_path):
    m = _tiny_clip("quick_gelu", 14, seed=3).float()
    m.save_pretrained(tmp_path)
    kw = tclip.read_config(str(tmp_path))
    assert kw == dict(img_size=56, patch_size=14, in_chans=3, num_classes=24, embed_dim=64, depth=3, num_heads=4,
                      mlp_ratio=2.0, eps_block=m.config.vision_config.layer_norm_eps,
                      eps_final=m.config.vision_config.layer_norm_eps, pre_norm=True, act="quick_gelu")
    sd, scale = tclip.engine_state_dict(tclip.load_weights(str(tmp_path)), kw["depth"])
    ref = m.state_dict()
    assert torch.equal(sd["blocks.1.attn.qkv.weight"], torch.cat([ref["vision_model.encoder.layers.1.self_attn.%s_proj.weight" % n]
                                                                  for n in "qkv"]))
    assert torch.equal(sd["head.weight"], ref["visual_projection.weight"])
    assert "patch_embed.proj.bias" not in sd and "head.bias" not in sd
    cfg = vit_config(**kw)
    names = [t[0] for t in _table(cfg)[0]]
    # every engine weight the table names is in the mapped checkpoint, but the two biases CLIP has not (read as zeros)
    assert set(names) - set(sd) == {"patch_embed.proj.bias", "head.bias"}


def save_tiny_clip_dir(path, act="quick_gelu", patch=14, seed=3):
    """A tiny CLIP checkpoint with a hand-written byte-level BPE vocabulary (every prompt of the tests tokenises) -> the model."""
    import json
    m = _tiny_clip(act, patch, seed).float()
    m.save_pretrained(path)
    merges = ["d o", "do g</w>", "c a", "ca t</w>", "p h", "ph o", "pho t", "phot o</w>", "o f</w>"]
    letters = sorted(set("adogctphf"))
    tokens = letters + [c + "</w>" for c in letters] + [m_.replace(" ", "") for m_ in merges]
    vocab = {t: i for i, t in enumerate(tokens + ["<|startoftext|>", "<|endoftext|>"])}
    assert len(vocab) < m.config.text_config.vocab_size
    with open(path / "vocab.json", "w") as f:
        json.dump(vocab, f)
    with open(path / "merges.txt", "w") as f:
        f.write("#version: 0.2\n" + "\n".join(merges) + "\n")
    return m


def test_encode_text_and_command_parsing(tmp_path):
    from transformer_explainability_b200 import clip_visualization as cv
    m = save_tiny_clip_dir(tmp_path)
    tower = tclip.text_tower(str(tmp_path))
    prompts = ["a dog", "a photo of a cat"]
    emb = tclip.encode_text(tower, prompts)
    assert emb.shape == (2, m.config.projection_dim)
    tok = tower[0]
    for p, e in zip(prompts, emb):
        ids = tok([p], return_tensors="pt")["input_ids"]
        assert tok.unk_token_id not in ids[0, 1:-1].tolist()
        with torch.no_grad():
            hidden = m.text_model(input_ids=ids).pooler_output
            assert torch.allclose(e, m.text_projection(hidden)[0], rtol=0, atol=1e-6)
    img = tmp_path / "imgs"
    img.mkdir()
    args = cv.parse_args(["--model-dir", str(tmp_path), "--images", str(img), "--text", "a dog", "a cat",
                          "--output-dir", str(tmp_path / "out"), "--start-layer", "1", "--batch-size", "4",
                          "--use-thresholding"])
    assert args.text == ["a dog", "a cat"] and args.start_layer == 1 and args.batch_size == 4 and args.use_thresholding
    for bad in (["--batch-size", "0"], ["--start-layer", "-1"]):
        with pytest.raises(SystemExit):
            cv.parse_args(["--model-dir", str(tmp_path), "--images", str(img), "--text", "a", "--output-dir", "o"] + bad)
    with pytest.raises(SystemExit):                 # no config.json
        cv.parse_args(["--model-dir", str(img), "--images", str(img), "--text", "a", "--output-dir", "o"])


GOLDEN = __import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "clip.npz")


def golden_model(z, key):
    """(engine state_dict fp32, heads, logit_scale, eps, act, images, text) of fixture model ``key`` ("t": the weights
    regenerated from the seed, ``oracle.make_golden_clip.tc_params``)."""
    if key == "t":
        from oracle.make_golden_clip import tc_params
        sd, heads = tc_params()
    else:
        sd, heads = {k[len(key) + 3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(key + ".w.")}, 4
    return (sd, heads, float(z[key + ".logit_scale"]), float(z[key + ".eps"]), {"q": "quick_gelu", "g": "gelu", "t": "quick_gelu"}[key],
            torch.from_numpy(z[key + ".images"]), torch.from_numpy(z[key + ".text"]))


@pytest.mark.parametrize("key", ["q", "g", "t"])
def test_oracle_against_fixture(key):
    """``oracle.clip`` in fp64 on the fixture's weights against what ``transformers`` computed (tests/golden/clip.npz)."""
    import numpy as np
    z = np.load(GOLDEN)
    sd, heads, scale, eps, act, x, text = golden_model(z, key)
    sd = {k: v.double() for k, v in sd.items()}
    attns, grads, s, _ = oclip.similarity_taps(sd, x.double(), heads, text.double(), scale, act=act, norm_eps=eps)
    ref_s = torch.from_numpy(z[key + ".hf.similarity"])
    assert torch.allclose(s, ref_s, rtol=1e-6, atol=0)
    for l, (a, g) in enumerate(zip(attns, grads)):
        ra, rg = torch.from_numpy(z["%s.hf.attn.%d" % (key, l)]), torch.from_numpy(z["%s.hf.grad.%d" % (key, l)])
        assert torch.allclose(a, ra, rtol=0, atol=1e-7)
        assert torch.allclose(g, rg, rtol=0, atol=1e-6 * rg.abs().max())
    for sl in (0, 1):
        ref = torch.from_numpy(z["%s.maps.sl%d" % (key, sl)])
        maps = agr.vit_map(attns, grads, sl, prefix=1)
        assert torch.allclose(maps, ref, rtol=0, atol=1e-6 * ref.abs().max())
