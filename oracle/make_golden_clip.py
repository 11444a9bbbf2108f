"""Generate ``tests/golden/clip.npz`` (TEST INFRASTRUCTURE, CPU).

    python -m oracle.make_golden_clip      # from the repo root

Two tiny random ``transformers.CLIPModel``s in fp64 with eager attention (vision tower: hidden 32, 3 layers, 4 heads,
MLP 64, projection 24; LayerNorm affines perturbed), ``q`` with QuickGELU at patch 14 on 56 x 56 images (N = 17) and
``g`` with GELU at patch 16 on 64 x 64 images (N = 17), a batch of 3 images with one text row each.  ``transformers``
gives the similarity (CLIP's ``logits_per_image`` of each pair), the attention probabilities (``output_attentions``) and
d s / d A (autograd through them); the maps are the unchanged ``oracle.attn_grad_rollout`` rule on those tensors.  Its
eager softmax runs in fp32 whatever the model's dtype, so the fixture pins the oracle to ~1e-8, not to fp64 rounding.

Keys (``{m}`` = ``q`` / ``g``): ``{m}.w.{name}`` the vision tower in the engine's names (``clip.engine_state_dict``; fp32,
the model's weights exactly),
``{m}.logit_scale`` (exp applied), ``{m}.eps``, ``{m}.images`` [3, 3, S, S], ``{m}.text`` [3, 24], ``{m}.hf.similarity`` [3],
``{m}.hf.attn.{l}`` / ``{m}.hf.grad.{l}`` [3, 4, 17, 17], ``{m}.maps.sl{0|1}`` [3, 16].

A third tower, ``t``, has the widths where the engine's tensor-core kernels apply (hidden 128, 2 heads of 64, MLP 512,
projection 128, 2 layers, QuickGELU, patch 14 on 56 x 56 images): its weights are ``tc_params()`` (``oracle.clip.init_params``,
regenerated from the seed, not stored), loaded into the ``transformers`` model; the keys are those above without ``t.w.*``
(and with 2 heads, 2 layers).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import attn_grad_rollout as agr    # noqa: E402
from oracle import clip as oclip               # noqa: E402
from transformer_explainability_b200 import clip as tclip    # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "clip.npz")
MODELS = {"q": ("quick_gelu", 14, 56, 2), "g": ("gelu", 16, 64, 1)}
TC = dict(img=56, patch=14, dim=128, depth=2, heads=2, mlp=512, embed=128, seed=4)


def tc_params():
    """The weights of tower ``t`` in the engine's names (fp32), and its heads."""
    return oclip.init_params(**TC)


def hf_state_dict(sd, depth, logit_scale):
    """The inverse of ``clip.engine_state_dict``: engine names -> ``CLIPModel``'s vision tower and projection keys."""
    v = "vision_model."
    D = sd["cls_token"].numel()
    hf = {v + "embeddings.patch_embedding.weight": sd["patch_embed.proj.weight"],
          v + "embeddings.class_embedding": sd["cls_token"].reshape(D),
          v + "embeddings.position_embedding.weight": sd["pos_embed"][0],
          v + "pre_layrnorm.weight": sd["norm_pre.weight"], v + "pre_layrnorm.bias": sd["norm_pre.bias"],
          v + "post_layernorm.weight": sd["norm.weight"], v + "post_layernorm.bias": sd["norm.bias"],
          "visual_projection.weight": sd["head.weight"], "logit_scale": torch.tensor(np.log(logit_scale))}
    for i in range(depth):
        h, e = v + "encoder.layers.%d." % i, "blocks.%d." % i
        for j, n in enumerate("qkv"):
            hf[h + "self_attn.%s_proj.weight" % n] = sd[e + "attn.qkv.weight"][j * D:(j + 1) * D]
            hf[h + "self_attn.%s_proj.bias" % n] = sd[e + "attn.qkv.bias"][j * D:(j + 1) * D]
        hf[h + "self_attn.out_proj.weight"], hf[h + "self_attn.out_proj.bias"] = sd[e + "attn.proj.weight"], sd[e + "attn.proj.bias"]
        for n, src in (("norm1", "layer_norm1"), ("norm2", "layer_norm2")):
            hf[h + src + ".weight"], hf[h + src + ".bias"] = sd[e + n + ".weight"], sd[e + n + ".bias"]
        for n in ("fc1", "fc2"):
            hf[h + "mlp.%s.weight" % n], hf[h + "mlp.%s.bias" % n] = sd[e + "mlp.%s.weight" % n], sd[e + "mlp.%s.bias" % n]
    return hf


def tc_clip():
    """The ``transformers.CLIPModel`` (fp64, eager) holding ``tc_params()``."""
    import transformers
    cfg = transformers.CLIPConfig(
        text_config=dict(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=2,
                         max_position_embeddings=16),
        vision_config=dict(hidden_size=TC["dim"], intermediate_size=TC["mlp"], num_hidden_layers=TC["depth"],
                           num_attention_heads=TC["heads"], image_size=TC["img"], patch_size=TC["patch"],
                           hidden_act="quick_gelu", layer_norm_eps=1e-5),
        projection_dim=TC["embed"])
    m = transformers.CLIPModel._from_config(cfg, attn_implementation="eager")
    sd, _ = tc_params()
    missing, unexpected = m.load_state_dict(hf_state_dict(sd, TC["depth"], 100.0), strict=False)
    assert not unexpected and all(k.startswith(("text_model.", "text_projection.")) or k.endswith("position_ids")
                                  for k in missing), missing
    return m.double().eval()


def tiny_clip(act, patch, img, seed):
    import transformers
    cfg = transformers.CLIPConfig(
        text_config=dict(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=2,
                         max_position_embeddings=16),
        vision_config=dict(hidden_size=32, intermediate_size=64, num_hidden_layers=3, num_attention_heads=4,
                           image_size=img, patch_size=patch, hidden_act=act),
        projection_dim=24)
    torch.manual_seed(seed)
    m = transformers.CLIPModel._from_config(cfg, attn_implementation="eager").double().eval()
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "layer_norm" in n or "layrnorm" in n:
                p.add_(0.1 * torch.randn_like(p))
    return m.float().double()                   # fp32-representable weights: the fixture stores them as fp32, exactly


def golden():
    out = {}
    for key, (act, patch, img, seed) in list(MODELS.items()) + [("t", ("quick_gelu", TC["patch"], TC["img"], TC["seed"]))]:
        m = tc_clip() if key == "t" else tiny_clip(act, patch, img, seed)
        vc = m.config.vision_config
        g = torch.Generator().manual_seed(5 + seed)
        x = torch.randn(3, 3, img, img, generator=g).double()            # fp32-representable: stored as fp32
        text = torch.randn(3, m.config.projection_dim, generator=g, dtype=torch.float64)
        sd, scale = tclip.engine_state_dict(m.state_dict(), vc.num_hidden_layers)
        with torch.enable_grad():
            o = m.vision_model(pixel_values=x, output_attentions=True)
            s = oclip.similarity(m.visual_projection(o.pooler_output), text, scale)
            grads = torch.autograd.grad(s.sum(), o.attentions)
        attns = [a.detach() for a in o.attentions]
        for n, v in sd.items():
            if key != "t":
                out["%s.w.%s" % (key, n)] = v.detach().float().numpy()
        out[key + ".logit_scale"] = np.float64(scale)
        out[key + ".eps"] = np.float64(vc.layer_norm_eps)
        out[key + ".images"] = x.float().numpy()
        out[key + ".text"] = text.numpy()
        out[key + ".hf.similarity"] = s.detach().numpy()
        for l, (a, gr) in enumerate(zip(attns, grads)):
            out["%s.hf.attn.%d" % (key, l)] = a.numpy()
            out["%s.hf.grad.%d" % (key, l)] = gr.numpy()
        for sl in (0, 1):
            out["%s.maps.sl%d" % (key, sl)] = agr.vit_map(attns, list(grads), sl, prefix=1).numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    golden()
