"""CLIP-architecture image towers (TEST INFRASTRUCTURE, CPU, any float dtype).

Restates the two ways a CLIP image tower (Hugging Face ``CLIPVisionModel`` + ``visual_projection``; timm's
``pre_norm=True`` ViTs) differs from the ViT of ``oracle.vit``:

* ``norm_pre``: a LayerNorm over the assembled tokens (cls + patches + pos_embed) before block 0 (CLIP's ``ln_pre``), at
  the blocks' epsilon;
* the MLP activation: erf GELU or QuickGELU, ``x * sigmoid(1.702 x)`` (CLIP's ``quick_gelu``);

and optional biases of the patch embedding and the head (CLIP has neither).  Everything downstream is ``oracle.vit``'s
wiring unchanged: inside ``architecture(act)`` its ``forward`` is this one, so ``oracle.vit.explain`` /
``explain_method`` (transformer_attribution, full, ...), ``oracle.alphabeta`` and ``oracle.attn_grad_rollout`` run on the
tower.  Both relevance rule libraries take LayerNorm and the activation as the identity, so no rule changes.

The image-text similarity is ``s = logit_scale * cos(x, t)`` of the projected image embedding x (the "logits": head
without bias) and a text embedding t, CLIP's ``logits_per_image``; its maps are the gradient-weighted attention rollout
of ``oracle.attn_grad_rollout`` with G_l = d s / d A_l.
"""
import contextlib

import torch
import torch.nn.functional as F

from . import attn_grad_rollout as agr
from . import vit as ovit


def quick_gelu(x):
    return x * torch.sigmoid(1.702 * x)


ACTS = {"gelu": F.gelu, "quick_gelu": quick_gelu}


def block_forward(p, cfg, i, t, act):
    """``oracle.vit.block_forward`` with the MLP activation ``act``."""
    pre = "blocks.%d." % i
    scale = (cfg.dim // cfg.heads) ** -0.5
    c = {"x_in": t}
    xn1 = F.layer_norm(t, (cfg.dim,), p[pre + "norm1.weight"], p[pre + "norm1.bias"], cfg.eps_block)
    qkv = F.linear(xn1, p[pre + "attn.qkv.weight"], p.get(pre + "attn.qkv.bias"))
    q, k, v = [ovit._split_heads(u, cfg.heads) for u in qkv.chunk(3, dim=-1)]
    attn = ((q @ k.transpose(-1, -2)) * scale).softmax(dim=-1)
    ctx = ovit._merge_heads(attn @ v)
    attn_out = F.linear(ctx, p[pre + "attn.proj.weight"], p[pre + "attn.proj.bias"])
    x_mid = t + attn_out
    xn2 = F.layer_norm(x_mid, (cfg.dim,), p[pre + "norm2.weight"], p[pre + "norm2.bias"], cfg.eps_block)
    g = ACTS[act](F.linear(xn2, p[pre + "mlp.fc1.weight"], p[pre + "mlp.fc1.bias"]))
    mlp_out = F.linear(g, p[pre + "mlp.fc2.weight"], p[pre + "mlp.fc2.bias"])
    c.update(xn1=xn1, q=q, k=k, v=v, attn=attn, ctx=ctx, attn_out=attn_out, x_mid=x_mid, xn2=xn2, g=g, mlp_out=mlp_out)
    return x_mid + mlp_out, c


def forward(params, x, num_heads, need_grad=False, norm_eps=None, act="gelu"):
    """``oracle.vit.forward`` of the tower: (logits [B,C] = the projected embedding for CLIP, cache).  The cache adds
    "x_pre" (the tokens entering block 0, after ``norm_pre`` when the params have it)."""
    cfg = ovit.ViTConfig(params, num_heads)
    if norm_eps is not None:
        cfg.eps_block = cfg.eps_final = norm_eps
    p = params
    B = x.shape[0]
    t = F.conv2d(x, p["patch_embed.proj.weight"], p.get("patch_embed.proj.bias"), stride=cfg.patch)
    t = torch.cat([p["cls_token"].expand(B, -1, -1), t.flatten(2).transpose(1, 2)], dim=1)
    tokens_pre_pos = t
    t = t + p["pos_embed"]
    if "norm_pre.weight" in p:
        t = F.layer_norm(t, (cfg.dim,), p["norm_pre.weight"], p["norm_pre.bias"], cfg.eps_block)
    if need_grad:
        t = t.detach().requires_grad_(True)
    cache = {"cfg": cfg, "blocks": [], "tokens_pre_pos": tokens_pre_pos.detach(), "image": x, "x_pre": t.detach()}
    for i in range(cfg.depth):
        t, c = block_forward(p, cfg, i, t, act)
        cache["blocks"].append(c)
    xf = F.layer_norm(t, (cfg.dim,), p["norm.weight"], p["norm.bias"], cfg.eps_final)
    cache["x_final_norm"] = xf
    cache["logits"] = F.linear(xf[:, 0], p["head.weight"], p.get("head.bias"))
    return cache["logits"], cache


@contextlib.contextmanager
def architecture(act="gelu"):
    """Inside the block, ``oracle.vit.forward`` is the tower's forward with activation ``act`` (norm_pre and the optional
    biases follow from the params), so every ``oracle.vit`` / ``alphabeta`` / ``attn_grad_rollout`` method runs on it."""
    saved = ovit.forward
    ovit.forward = lambda params, x, num_heads, need_grad=False, norm_eps=None: forward(params, x, num_heads, need_grad,
                                                                                        norm_eps, act)
    try:
        yield
    finally:
        ovit.forward = saved


def similarity(image_embeds, text, logit_scale):
    """CLIP's logits_per_image of each image with its own text row: logit_scale * cos(x_b, t_b) -> [B]."""
    return logit_scale * (image_embeds * text).sum(-1) / (image_embeds.norm(dim=-1) * text.norm(dim=-1))


def similarity_taps(params, x, num_heads, text, logit_scale, act="quick_gelu", norm_eps=1e-5):
    """(attns, grads = d s / d A_l, s [B], cache) of the tower's forward on images x with text rows text [B, E]."""
    with torch.enable_grad():
        logits, cache = forward(params, x, num_heads, need_grad=True, norm_eps=norm_eps, act=act)
        s = similarity(logits, text.to(logits.dtype), logit_scale)
        attns = [c["attn"] for c in cache["blocks"]]
        grads = torch.autograd.grad(s.sum(), attns)
    return [a.detach() for a in attns], [g.detach() for g in grads], s.detach(), cache


def explain_similarity(params, x, num_heads, text, logit_scale, start_layer=0, act="quick_gelu", norm_eps=1e-5):
    """The gradient-weighted attention rollout of the similarity: (maps [B, N-1], s [B])."""
    attns, grads, s, _ = similarity_taps(params, x, num_heads, text, logit_scale, act, norm_eps)
    with torch.no_grad():
        return agr.vit_map(attns, grads, start_layer, prefix=1), s


def init_params(img=224, patch=16, dim=768, depth=12, heads=12, mlp=3072, embed=512, seed=0, dtype=torch.float32,
                pre_norm=True, biases=False):
    """Random CLIP-like tower weights in the engine's names (``oracle.vit.init_params`` with ``rand_affine``, plus
    ``norm_pre``; without ``biases`` no patch-embedding or head bias, as CLIP).  head = the visual projection [embed, dim]."""
    p, _ = ovit.init_params("vit_tiny_test", seed=seed, rand_affine=True, img=img, patch=patch, dim=dim, depth=depth,
                            heads=heads, mlp=mlp, classes=embed)
    g = torch.Generator().manual_seed(seed + 7919)
    if pre_norm:
        p["norm_pre.weight"] = 1 + 0.2 * torch.randn(dim, generator=g)
        p["norm_pre.bias"] = 0.05 * torch.randn(dim, generator=g)
    # CLIP's class and position embeddings are O(1) before ln_pre (scale dim^-0.5 * N(0, 1)); ln_pre normalises them
    p["cls_token"] = p["cls_token"] * 20
    p["pos_embed"] = p["pos_embed"] * 20
    if not biases:
        del p["patch_embed.proj.bias"], p["head.bias"]
    return {k: v.to(dtype) for k, v in p.items()}, heads
