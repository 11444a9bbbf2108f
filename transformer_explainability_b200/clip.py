"""Explain CLIP image encoders on the engine: which patches make an image match a text.

A CLIP image tower is the engine's ViT with a LayerNorm before block 0 (``ln_pre``), QuickGELU (or GELU) MLPs, no patch
or head bias, and the visual projection as the "head": the engine's logits are the projected image embedding x.  The
similarity to a text embedding t is CLIP's ``logits_per_image``, s = exp(logit_scale) * cos(x, t); the explanation is
the gradient-weighted attention rollout (Chefer, Gur, Wolf, ICCV 2021) of s, started from d s / d x
(``te_vit_similarity_seed``, ``TE_FLAG_SIMILARITY_SEED``).

``CLIPExplainer`` loads a local Hugging Face CLIP directory (``config.json`` with ``model_type: "clip"``, the weights
in ``model.safetensors`` or ``pytorch_model.bin``).  The text tower runs in torch through ``transformers``
(``encode_text``): images are the engine's batch dimension, a prompt is one [E] vector.
"""
import math
import os

import torch

from . import _lib
from .engine import ViTEngine, vit_config

_ACTS = {"quick_gelu": "quick_gelu", "gelu": "gelu"}


def read_config(model_dir):
    """The vision tower of a Hugging Face CLIP directory as ``vit_config`` arguments (and the projection width)."""
    from transformers import CLIPConfig
    cfg = CLIPConfig.from_pretrained(model_dir)
    if cfg.model_type != "clip":
        raise ValueError("%s: model_type %r, expected 'clip'" % (model_dir, cfg.model_type))
    v = cfg.vision_config
    if v.hidden_act not in _ACTS:
        raise ValueError("%s: hidden_act %r is not one the engine runs (quick_gelu, gelu)" % (model_dir, v.hidden_act))
    return dict(img_size=v.image_size, patch_size=v.patch_size, in_chans=getattr(v, "num_channels", 3),
                num_classes=cfg.projection_dim, embed_dim=v.hidden_size, depth=v.num_hidden_layers,
                num_heads=v.num_attention_heads, mlp_ratio=v.intermediate_size / v.hidden_size, eps_block=v.layer_norm_eps,
                eps_final=v.layer_norm_eps, pre_norm=True, act=_ACTS[v.hidden_act])


def engine_state_dict(hf, depth):
    """Hugging Face ``CLIPModel`` keys -> the engine's ViT names: q / k / v into ``qkv``, ``pre_layrnorm`` -> ``norm_pre``,
    ``post_layernorm`` -> ``norm``, ``visual_projection`` -> ``head``.  Returns (state_dict, exp(logit_scale))."""
    v = "vision_model."
    D = hf[v + "embeddings.class_embedding"].numel()
    sd = {"patch_embed.proj.weight": hf[v + "embeddings.patch_embedding.weight"],
          "cls_token": hf[v + "embeddings.class_embedding"].reshape(1, 1, D),
          "pos_embed": hf[v + "embeddings.position_embedding.weight"].unsqueeze(0),
          "norm_pre.weight": hf[v + "pre_layrnorm.weight"], "norm_pre.bias": hf[v + "pre_layrnorm.bias"],
          "norm.weight": hf[v + "post_layernorm.weight"], "norm.bias": hf[v + "post_layernorm.bias"],
          "head.weight": hf["visual_projection.weight"]}
    for i in range(depth):
        h, e = v + "encoder.layers.%d." % i, "blocks.%d." % i
        a = h + "self_attn."
        sd[e + "attn.qkv.weight"] = torch.cat([hf[a + n + "_proj.weight"] for n in "qkv"])
        sd[e + "attn.qkv.bias"] = torch.cat([hf[a + n + "_proj.bias"] for n in "qkv"])
        sd[e + "attn.proj.weight"], sd[e + "attn.proj.bias"] = hf[a + "out_proj.weight"], hf[a + "out_proj.bias"]
        for n in ("norm1", "norm2"):
            src = h + ("layer_norm1." if n == "norm1" else "layer_norm2.")
            sd[e + n + ".weight"], sd[e + n + ".bias"] = hf[src + "weight"], hf[src + "bias"]
        for n in ("fc1", "fc2"):
            sd[e + "mlp." + n + ".weight"], sd[e + "mlp." + n + ".bias"] = hf[h + "mlp." + n + ".weight"], hf[h + "mlp." + n + ".bias"]
    return sd, math.exp(float(hf["logit_scale"]))


def load_weights(model_dir):
    """The checkpoint's tensors (``model.safetensors`` or ``pytorch_model.bin``)."""
    st = os.path.join(model_dir, "model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file
        return load_file(st)
    return torch.load(os.path.join(model_dir, "pytorch_model.bin"), map_location="cpu", weights_only=True)


class CLIPExplainer:
    """The CLIP image tower of ``model_dir`` on the engine.  flags: the engine's kernel selection (the method flags are
    added per call)."""

    def __init__(self, model_dir, device=None, flags=_lib.FLAG_BENCH_DEFAULT):
        self.model_dir = model_dir
        self.kwargs = read_config(model_dir)
        sd, self.logit_scale = engine_state_dict(load_weights(model_dir), self.kwargs["depth"])
        self.engine = ViTEngine(vit_config(**self.kwargs), sd, device=device, flags=flags)
        self.grid = self.kwargs["img_size"] // self.kwargs["patch_size"]
        self._text = None

    def generate_attn_grad_rollout(self, images, text_features, start_layer=0):
        """images [B, 3, H, W] (CLIP-normalised), text_features [B, E] (one per image) or [E] -> (maps [B, N-1] on the patch
        grid, similarity [B] = CLIP's logits_per_image of each pair)."""
        self.engine.forward(images)
        return self.explain_forwarded(text_features, start_layer)

    def explain_forwarded(self, text_features, start_layer=0):
        """The maps and similarities of the images of the last ``engine.forward`` with another text: one seed launch and one
        ``attribute``, the forward is not repeated."""
        sim = self.engine.similarity(text_features, self.logit_scale)
        maps, _ = self.engine.attribute(start_layer=start_layer, similarity_seeded=True)
        return maps, sim

    def encode_text(self, prompts):
        """prompts (list of str) -> text embeddings [P, E] from the checkpoint's text tower (``encode_text``)."""
        if self._text is None:
            self._text = text_tower(self.model_dir)
        return encode_text(self._text, prompts)


def text_tower(model_dir):
    """(tokenizer, CLIPModel) of the checkpoint, for ``encode_text`` (torch, fp32, on the host)."""
    from transformers import CLIPModel, CLIPTokenizer
    return CLIPTokenizer.from_pretrained(model_dir), CLIPModel.from_pretrained(model_dir, dtype=torch.float32).eval()


@torch.no_grad()
def encode_text(tower, prompts):
    """prompts (list of str) -> ``get_text_features`` [P, E], one prompt at a time (no padding enters the causal tower)."""
    tok, model = tower
    out = []
    for p in prompts:
        ids = tok([p], return_tensors="pt")
        t = model.get_text_features(input_ids=ids["input_ids"], attention_mask=ids["attention_mask"])
        out.append((t if torch.is_tensor(t) else t.pooler_output)[0])
    return torch.stack(out)
