"""ViT transformer-attribution oracle (TEST INFRASTRUCTURE, CPU, any float dtype).

Restates the wiring of ``/root/reference/baselines/ViT/ViT_LRP.py`` on top of
``oracle.rules``:

* forward           ``VisionTransformer.forward`` ``:305-322``, ``Block.forward`` ``:196-201``,
                    ``Attention.forward`` ``:132-152``, ``Mlp.forward`` ``:61-67``, ``PatchEmbed`` ``:230-236``
* attention grads   what ``attn.register_hook(self.save_attn_gradients)`` ``:145`` captures
                    when ``ViT_explanation_generator.py:31-38`` back-propagates the one-hot
* relprop           ``VisionTransformer.relprop`` ``:324-369``, ``Block.relprop`` ``:203-213``,
                    ``Attention.relprop`` ``:154-177``, ``Mlp.relprop`` ``:69-74``
* rollout           ``compute_rollout_attention`` ``:38-49`` and ``rollout[:, 0, 1:]`` ``:368``

``params`` is a dict keyed like the reference ``state_dict`` (timm names).  An
optional ``dist_token`` / ``head_dist.*`` pair switches on the 198-token
distilled-DeiT extension (SURVEY.md §7f; not in the reference — "oracle-extended").
A batch is a set of independent B=1 explanations (per-sample reductions).
"""
import math
import torch
import torch.nn.functional as F

from . import rules


class ViTConfig:
    def __init__(self, params, num_heads):
        self.dim = params["pos_embed"].shape[-1]
        self.tokens = params["pos_embed"].shape[1]
        self.patch = params["patch_embed.proj.weight"].shape[-1]
        self.in_chans = params["patch_embed.proj.weight"].shape[1]
        self.depth = 1 + max(int(k.split(".")[1]) for k in params if k.startswith("blocks."))
        self.heads = num_heads
        self.mlp_dim = params["blocks.0.mlp.fc1.weight"].shape[0]
        self.num_classes = params["head.weight"].shape[0]
        self.distilled = "dist_token" in params
        self.eps_block = 1e-6      # ViT_LRP.py:184,187
        self.eps_final = 1e-5      # ViT_LRP.py:266 (nn.LayerNorm default)


def _split_heads(t, h):
    b, n, d = t.shape
    return t.reshape(b, n, h, d // h).permute(0, 2, 1, 3)       # 'b n (h d) -> b h n d'


def _merge_heads(t):
    b, h, n, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(b, n, h * d)           # 'b h n d -> b n (h d)'


def block_forward(p, cfg, i, t):
    """``Block.forward`` (``:196-201``) of block ``i`` on its input ``t`` [B,N,D]: returns (output, the block's cache)."""
    pre = "blocks.%d." % i
    scale = (cfg.dim // cfg.heads) ** -0.5
    c = {"x_in": t}
    xn1 = F.layer_norm(t, (cfg.dim,), p[pre + "norm1.weight"], p[pre + "norm1.bias"], cfg.eps_block)
    qkv = F.linear(xn1, p[pre + "attn.qkv.weight"], p.get(pre + "attn.qkv.bias"))
    q, k, v = [_split_heads(u, cfg.heads) for u in qkv.chunk(3, dim=-1)]   # '(qkv h d)'
    dots = (q @ k.transpose(-1, -2)) * scale
    attn = dots.softmax(dim=-1)
    ctx = _merge_heads(attn @ v)
    attn_out = F.linear(ctx, p[pre + "attn.proj.weight"], p[pre + "attn.proj.bias"])
    x_mid = t + attn_out
    xn2 = F.layer_norm(x_mid, (cfg.dim,), p[pre + "norm2.weight"], p[pre + "norm2.bias"], cfg.eps_block)
    hpre = F.linear(xn2, p[pre + "mlp.fc1.weight"], p[pre + "mlp.fc1.bias"])
    g = F.gelu(hpre)
    mlp_out = F.linear(g, p[pre + "mlp.fc2.weight"], p[pre + "mlp.fc2.bias"])
    c.update(xn1=xn1, q=q, k=k, v=v, attn=attn, ctx=ctx, attn_out=attn_out, x_mid=x_mid,
             xn2=xn2, g=g, mlp_out=mlp_out)
    return x_mid + mlp_out, c


def forward(params, x, num_heads, need_grad=False, norm_eps=None):
    """Returns (logits [B,C], cache).  ``cache`` holds every tensor the relprop needs.
    ``norm_eps``: one epsilon for every LayerNorm (the ``ViT_new`` factories, ``ViT_new.py:226-254``)."""
    cfg = ViTConfig(params, num_heads)
    if norm_eps is not None:
        cfg.eps_block = cfg.eps_final = norm_eps
    p = params
    B = x.shape[0]
    t = F.conv2d(x, p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], stride=cfg.patch)
    t = t.flatten(2).transpose(1, 2)
    toks = [p["cls_token"].expand(B, -1, -1)]
    if cfg.distilled:
        toks.append(p["dist_token"].expand(B, -1, -1))
    t = torch.cat(toks + [t], dim=1)
    tokens_pre_pos = t
    t = t + p["pos_embed"]
    if need_grad:
        t = t.detach().requires_grad_(True)     # puts every attn tensor on an autograd graph
    cache = {"cfg": cfg, "blocks": [], "tokens_pre_pos": tokens_pre_pos.detach(), "image": x}
    for i in range(cfg.depth):
        t, c = block_forward(p, cfg, i, t)
        cache["blocks"].append(c)
    xf = F.layer_norm(t, (cfg.dim,), p["norm.weight"], p["norm.bias"], cfg.eps_final)
    cache["x_final_norm"] = xf
    pooled = xf[:, 0]
    logits = F.linear(pooled, p["head.weight"], p["head.bias"])
    if cfg.distilled:
        logits_d = F.linear(xf[:, 1], p["head_dist.weight"], p["head_dist.bias"])
        logits = (logits + logits_d) / 2
    cache["logits"] = logits
    return logits, cache


def attention_gradients(cache, seed):
    """d(sum(seed*logits))/d attn_l for every block: list of [B,H,N,N]."""
    loss = (seed * cache["logits"]).sum()
    attns = [c["attn"] for c in cache["blocks"]]
    return list(torch.autograd.grad(loss, attns, retain_graph=True))


def relprop(params, cache, seed, start_layer=0, taps=None, to_input=False, variant="ours"):
    """LRP pass; returns list (per block) of attn_cam [B,H,N,N] (``ViT_LRP.py:165``).
    ``variant="lrp"``: the rule library of ``modules/layers_lrp.py`` (``baselines/ViT/ViT_orig_LRP.py``: Linear with
    separate denominators, Add without ratio normalisation) instead of ``modules/layers_ours.py``.

    Blocks below ``start_layer`` are never consumed by the rollout and are returned as None.
    ``to_input=True`` runs every block to its end (what the reference always does, ``:331-332``) and
    returns ``(cams, r)`` with ``r`` the relevance at the encoder input [B,N,D].
    """
    cfg = cache["cfg"]
    p = params
    xf = cache["x_final_norm"]
    lin = rules.linear_relprop_lrp if variant == "lrp" else rules.linear_relprop
    add = rules.add_relprop_simple if variant == "lrp" else rules.add_relprop
    # head.relprop -> unsqueeze -> pool.relprop (IndexSelect) -> norm.relprop (identity)  :327-330
    if cfg.distilled:
        # extension: averaged logits = Add of two halves; seed relevance split evenly through both heads
        r_cls = lin(xf[:, 0], p["head.weight"], seed / 2)
        r_dst = lin(xf[:, 1], p["head_dist.weight"], seed / 2)
        r = rules.index_select_relprop(xf, r_cls.unsqueeze(1), 0) + \
            rules.index_select_relprop(xf, r_dst.unsqueeze(1), 1)
    else:
        r_cls = lin(xf[:, 0], p["head.weight"], seed)
        r = rules.index_select_relprop(xf, r_cls.unsqueeze(1), 0)
    cams = [None] * cfg.depth
    for i in reversed(range(max(start_layer, 0), cfg.depth)):
        pre = "blocks.%d." % i
        c = cache["blocks"][i]
        t = {} if taps is not None else None
        if t is not None:
            taps[i] = t
            t["r_in"] = r
        # Block.relprop :203-213
        r1, r2 = add(c["x_mid"], c["mlp_out"], r)                 # add2
        if t is not None:
            t["add2_r1"], t["add2_r2"] = r1, r2
        r2 = lin(c["g"], p[pre + "mlp.fc2.weight"], r2)        # fc2 ; GELU identity
        if t is not None:
            t["fc2"] = r2
        r2 = lin(c["xn2"], p[pre + "mlp.fc1.weight"], r2)      # fc1 ; norm2 identity
        if t is not None:
            t["fc1"] = r2
        r = rules.clone_relprop(c["x_mid"], (r1, r2))                           # clone2
        if t is not None:
            t["clone2"] = r
        r1, r2 = add(c["x_in"], c["attn_out"], r)                 # add1
        if t is not None:
            t["add1_r1"], t["add1_r2"] = r1, r2
        # Attention.relprop :154-177
        r2 = lin(c["ctx"], p[pre + "attn.proj.weight"], r2)
        if t is not None:
            t["proj"] = r2
        r2 = _split_heads(r2, cfg.heads)
        cam1, cam_v = rules.matmul_av_relprop(c["attn"], c["v"], r2)
        cam1 = cam1 / 2
        cam_v = cam_v / 2
        cams[i] = cam1                                                          # save_attn_cam :165
        if i == start_layer and not to_input:
            break                                                               # nothing below is consumed
        cam_q, cam_k = rules.matmul_qk_relprop(c["q"], c["k"], cam1)
        cam_q = cam_q / 2
        cam_k = cam_k / 2
        r_qkv = torch.cat([_merge_heads(cam_q), _merge_heads(cam_k), _merge_heads(cam_v)], dim=-1)
        r2 = lin(c["xn1"], p[pre + "attn.qkv.weight"], r_qkv)  # norm1 identity
        r = rules.clone_relprop(c["x_in"], (r1, r2))                            # clone1
        if t is not None:
            t["r_qkv"], t["qkv"], t["clone1"] = r_qkv, r2, r
    if to_input:
        return cams, r
    return cams


METHODS = ("transformer_attribution", "grad", "rollout", "full", "last_layer", "last_layer_attn", "second_layer")


def explain_method(params, x, num_heads, method, index=None, start_layer=0, is_ablation=False, variant="ours"):
    """``LRP.generate_LRP(method=...)`` for every branch of ``VisionTransformer.relprop``
    (``ViT_LRP.py:337-398``), batch = independent B=1 explanations.  Returns (map, index):
    [B,N-1] for the token methods, [B,H,W] for ``full`` (relevance of every pixel, channels summed)."""
    if method in ("transformer_attribution", "grad"):
        return explain(params, x, num_heads, index=index, start_layer=start_layer, variant=variant)
    with torch.enable_grad():
        logits, cache = forward(params, x, num_heads, need_grad=True)
        if index is None:
            index = logits.argmax(dim=-1)
        index = torch.as_tensor(index).reshape(-1).long()
        seed = torch.zeros_like(logits)
        seed[torch.arange(logits.shape[0]), index] = 1
        grads = attention_gradients(cache, seed)
    cfg = cache["cfg"]
    first = 2 if cfg.distilled else 1
    with torch.no_grad():
        cache_d = {"cfg": cfg, "x_final_norm": cache["x_final_norm"].detach(),
                   "blocks": [{k: v.detach() for k, v in c.items()} for c in cache["blocks"]]}
        cams, r = relprop(params, cache_d, seed, 0, to_input=True, variant=variant)
        if method == "full":                                                    # :337-343
            pos = params["pos_embed"].expand_as(cache["tokens_pre_pos"])
            r, _ = (rules.add_relprop_simple if variant == "lrp" else rules.add_relprop)(cache["tokens_pre_pos"], pos, r)
            r = r[:, first:]
            g = x.shape[-1] // cfg.patch
            r = r.transpose(1, 2).reshape(r.shape[0], cfg.dim, x.shape[-2] // cfg.patch, g)   # PatchEmbed.relprop :238-242
            r = rules.conv_zb_relprop(x, params["patch_embed.proj.weight"], r, cfg.patch)
            return r.sum(dim=1), index
        if method == "rollout":                                                 # :345-354
            mats = [c.clamp(min=0).mean(dim=1) for c in cams]
            return rules.rollout(mats, start_layer=start_layer)[:, 0, first:], index
        if method in ("last_layer", "second_layer"):                            # :371-380, :389-398
            l = cfg.depth - 1 if method == "last_layer" else 1
            c = cams[l]
            if is_ablation:
                c = grads[l] * c
            return c.clamp(min=0).mean(dim=1)[:, 0, first:], index
        if method == "last_layer_attn":                                         # :382-387
            return cache_d["blocks"][-1]["attn"].clamp(min=0).mean(dim=1)[:, 0, first:], index
    raise ValueError("unknown method %r" % (method,))


def explain(params, x, num_heads, index=None, start_layer=0, return_taps=False, variant="ours"):
    """``LRP.generate_LRP(method='transformer_attribution')`` for a batch of independent
    samples.  Returns (maps [B,N-1(-1 if distilled)], index [B]) (+ taps)."""
    with torch.enable_grad():
        logits, cache = forward(params, x, num_heads, need_grad=True)
        if index is None:
            index = logits.argmax(dim=-1)
        index = torch.as_tensor(index).reshape(-1).long()
        seed = torch.zeros_like(logits)
        seed[torch.arange(logits.shape[0]), index] = 1
        grads = attention_gradients(cache, seed)
    with torch.no_grad():
        cache_d = {"cfg": cache["cfg"], "x_final_norm": cache["x_final_norm"].detach(),
                   "blocks": [{k: v.detach() for k, v in c.items()} for c in cache["blocks"]]}
        rtaps = {} if return_taps else None
        cams = relprop(params, cache_d, seed, start_layer, taps=rtaps, variant=variant)
        mats = [rules.aggregate(g, c) if c is not None else torch.zeros_like(g[:, 0])
                for g, c in zip(grads, cams)]
        joint = rules.rollout(mats, start_layer=start_layer, normalize=False)
        first = 2 if cache["cfg"].distilled else 1
        out = joint[:, 0, first:]
    if return_taps:
        return out, index, {"logits": logits.detach(), "grads": grads, "cams": cams, "mats": mats,
                            "joint": joint, "cache": cache_d, "relprop": rtaps}
    return out, index


def init_params(cfg_name="vit_base_patch16_224", seed=0, dtype=torch.float32, **over):
    """Deterministic random-init parameters with the reference's state_dict keys and
    init distributions (``ViT_LRP.py:276-299``: trunc_normal(std=.02) Linear / pos / cls,
    LayerNorm 1/0, zero biases; conv keeps torch's default init).  Used wherever the
    reference itself is not importable (GPU box)."""
    presets = {
        "vit_base_patch16_224": dict(img=224, patch=16, dim=768, depth=12, heads=12, mlp=3072, classes=1000),
        "vit_large_patch16_224": dict(img=224, patch=16, dim=1024, depth=24, heads=16, mlp=4096, classes=1000),
        "deit_base_patch16_224": dict(img=224, patch=16, dim=768, depth=12, heads=12, mlp=3072, classes=1000),
        "deit_base_distilled_patch16_224": dict(img=224, patch=16, dim=768, depth=12, heads=12, mlp=3072,
                                                classes=1000, distilled=True),
        "vit_tiny_test": dict(img=32, patch=8, dim=64, depth=3, heads=4, mlp=256, classes=10),
    }
    c = dict(presets[cfg_name])
    c.update(over)
    g = torch.Generator().manual_seed(seed)

    def tn(*shape):
        t = torch.empty(*shape)
        torch.nn.init.trunc_normal_(t, std=.02, a=-2., b=2., generator=g)
        return t

    D, P = c["dim"], c["patch"]
    ntok = (c["img"] // P) ** 2 + (2 if c.get("distilled") else 1)
    p = {}
    fan_in = 3 * P * P
    bound = 1 / math.sqrt(fan_in)
    p["patch_embed.proj.weight"] = (torch.rand(D, 3, P, P, generator=g) * 2 - 1) * bound
    p["patch_embed.proj.bias"] = (torch.rand(D, generator=g) * 2 - 1) * bound
    p["cls_token"] = tn(1, 1, D)
    if c.get("distilled"):
        p["dist_token"] = tn(1, 1, D)
    p["pos_embed"] = tn(1, ntok, D)
    for i in range(c["depth"]):
        pre = "blocks.%d." % i
        p[pre + "norm1.weight"] = torch.ones(D)
        p[pre + "norm1.bias"] = torch.zeros(D)
        p[pre + "attn.qkv.weight"] = tn(3 * D, D)
        p[pre + "attn.qkv.bias"] = torch.zeros(3 * D)
        p[pre + "attn.proj.weight"] = tn(D, D)
        p[pre + "attn.proj.bias"] = torch.zeros(D)
        p[pre + "norm2.weight"] = torch.ones(D)
        p[pre + "norm2.bias"] = torch.zeros(D)
        p[pre + "mlp.fc1.weight"] = tn(c["mlp"], D)
        p[pre + "mlp.fc1.bias"] = torch.zeros(c["mlp"])
        p[pre + "mlp.fc2.weight"] = tn(D, c["mlp"])
        p[pre + "mlp.fc2.bias"] = torch.zeros(D)
    p["norm.weight"] = torch.ones(D)
    p["norm.bias"] = torch.zeros(D)
    p["head.weight"] = tn(c["classes"], D)
    p["head.bias"] = torch.zeros(c["classes"])
    if c.get("distilled"):
        p["head_dist.weight"] = tn(c["classes"], D)
        p["head_dist.bias"] = torch.zeros(c["classes"])
    if c.get("rand_affine"):
        # pretrained-like: non-trivial biases and LayerNorm affine so those paths are exercised
        for k in sorted(p):
            if k.endswith("norm1.weight") or k.endswith("norm2.weight") or k == "norm.weight":
                p[k] = 1 + 0.2 * torch.randn(p[k].shape, generator=g)
            elif k.endswith(".bias") and not k.startswith("patch_embed"):
                p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
    return {k: v.to(dtype) for k, v in p.items()}, c["heads"]


def baseline_rollout(params, x, num_heads, start_layer=0, norm_eps=1e-6):
    """``Baselines.generate_rollout`` (``ViT_explanation_generator.py:73-83``) on the hook-free ``ViT_new`` model:
    head-averaged raw attention of every block -> the file's own ROW-NORMALISED rollout (``:7-18``) -> [B,N-1]."""
    with torch.no_grad():
        _, cache = forward(params, x, num_heads, norm_eps=norm_eps)
        mats = [c["attn"].mean(dim=1) for c in cache["blocks"]]
        return rules.rollout(mats, start_layer=start_layer, normalize=True)[:, 0, 1:]


def baseline_cam_attn(params, x, num_heads, index=None, norm_eps=1e-6):
    """``Baselines.generate_cam_attn`` (``:50-71``): CLS row of the last block's attention weighted per head by the
    mean (over the patch positions) of its class gradient, relu(mean over heads), min-max normalised -> [B,g,g]."""
    with torch.enable_grad():
        logits, cache = forward(params, x, num_heads, need_grad=True, norm_eps=norm_eps)
        if index is None:
            index = logits.argmax(dim=-1)
        index = torch.as_tensor(index).reshape(-1).long()
        seed = torch.zeros_like(logits)
        seed[torch.arange(logits.shape[0]), index] = 1
        grad = attention_gradients(cache, seed)[-1]
    with torch.no_grad():
        cam = cache["blocks"][-1]["attn"].detach()[:, :, 0, 1:]               # [B,H,np]
        g = grad[:, :, 0, 1:].mean(dim=2, keepdim=True)
        cam = (cam * g).mean(dim=1).clamp(min=0)
        lo = cam.amin(dim=1, keepdim=True)
        hi = cam.amax(dim=1, keepdim=True)
        cam = (cam - lo) / (hi - lo)
        side = int(round(cam.shape[1] ** 0.5))
        return cam.reshape(-1, side, side), index
