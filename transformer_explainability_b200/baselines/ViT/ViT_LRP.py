"""Drop-in for the reference's ``baselines/ViT/ViT_LRP.py``.

Same public surface — ``VisionTransformer`` (same constructor arguments and ``state_dict`` keys),
``vit_base_patch16_224`` / ``vit_large_patch16_224`` / ``deit_base_patch16_224`` factories,
``compute_rollout_attention``, ``model(x)`` and ``model.relprop(cam, method=..., start_layer=..., alpha=1)``,
``blk.attn.get_attn() / get_attn_gradients() / get_attn_cam()`` — but the model is a parameter
container: ``forward`` and ``relprop`` are executed by the CUDA engine (``engine.ViTEngine``) behind the
C ABI, for a whole batch of independent inputs at once.  No autograd graph, no hooks, no ``param.grad``
side effect (documented deviation, SURVEY.md §8b).

``deit_base_distilled_patch16_224`` (198 tokens, dist token + second head) is an extension that the
reference does not contain (SURVEY.md §7f).
"""
import weakref

import torch
import torch.nn as nn

from transformer_explainability_b200 import ops
from transformer_explainability_b200 import _lib
from transformer_explainability_b200.engine import ViTEngine, vit_config

__all__ = ["VisionTransformer", "compute_rollout_attention", "vit_base_patch16_224", "vit_large_patch16_224",
           "deit_base_patch16_224", "deit_base_distilled_patch16_224"]


def compute_rollout_attention(all_layer_matrices, start_layer=0):
    """``ViT_LRP.py:38-49``: (M_i + I) chained from ``start_layer``; list of [B,N,N] -> [B,N,N]."""
    return ops.compute_rollout_attention(all_layer_matrices, start_layer=start_layer, normalize=False)


class _AttentionView(nn.Module):
    """Parameter holder for ``blocks[i].attn`` + the accessors of ``ViT_LRP.py:102-130`` served from the
    engine workspace (valid after ``model(x)`` / ``model.relprop(...)`` of the owning model)."""

    def __init__(self, dim, num_heads, qkv_bias):
        super().__init__()
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self._owner = None
        self._layer = -1

    def _t(self, name):
        owner = self._owner() if self._owner is not None else None
        if owner is None:
            raise RuntimeError("this attention view's model no longer exists")
        return owner._engine_tensor(name, self._layer)

    def __getstate__(self):                    # the back-reference is re-made by the owning model's __setstate__
        state = self.__dict__.copy()
        state["_owner"] = None
        return state

    def get_attn(self):
        return self._t("attn")

    def get_attention_map(self):               # ViT_new.py's name for the same probabilities
        return self._t("attn")

    def get_attn_cam(self):
        return self._t("attn_cam")

    def get_attn_gradients(self):
        return self._t("attn_grad")

    def get_v(self):
        qkv = self._t("qkv")                                  # [B,N,3D]  '(qkv h d)'
        b, n, d3 = qkv.shape
        d = d3 // 3
        return qkv[:, :, 2 * d:].reshape(b, n, self.num_heads, d // self.num_heads).permute(0, 2, 1, 3)


class _Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


class _Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio, qkv_bias):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = _AttentionView(dim, num_heads, qkv_bias)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = _Mlp(dim, int(dim * mlp_ratio))


class _PatchEmbed(nn.Module):
    def __init__(self, img_size, patch_size, in_chans, embed_dim):
        super().__init__()
        self.img_size = (img_size, img_size)
        self.patch_size = (patch_size, patch_size)
        self.num_patches = (img_size // patch_size) ** 2
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)


class VisionTransformer(nn.Module):
    """``ViT_LRP.py:247-398`` re-hosted on the CUDA engine."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, num_classes=1000, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4., qkv_bias=False, mlp_head=False, drop_rate=0., attn_drop_rate=0.,
                 distilled=False, norm_eps=None, pre_norm=False, act_layer="gelu"):
        """pre_norm / act_layer: the CLIP-architecture image towers (timm ``pre_norm=True``): a LayerNorm ``norm_pre`` over
        the assembled tokens before block 0 (the blocks' epsilon), and the MLP activation "gelu" (erf) or "quick_gelu"
        (x * sigmoid(1.702 x)).  Both relevance rule libraries take LayerNorm and the activation as the identity."""
        super().__init__()
        if mlp_head:
            raise NotImplementedError("mlp_head=True is not used by any reference factory")
        self.num_classes = num_classes
        self.num_features = self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.distilled = bool(distilled)
        self.patch_embed = _PatchEmbed(img_size, patch_size, in_chans, embed_dim)
        n_tok = self.patch_embed.num_patches + (2 if distilled else 1)
        self.pos_embed = nn.Parameter(torch.zeros(1, n_tok, embed_dim))
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        if distilled:
            self.dist_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        if pre_norm:
            self.norm_pre = nn.LayerNorm(embed_dim, eps=1e-6)
        self.blocks = nn.ModuleList([_Block(embed_dim, num_heads, mlp_ratio, qkv_bias) for _ in range(depth)])
        self.norm = nn.LayerNorm(embed_dim)
        if norm_eps is not None:               # ViT_new passes one norm_layer (one epsilon) to every LayerNorm
            self.norm.eps = norm_eps
            for blk in self.blocks:
                blk.norm1.eps = blk.norm2.eps = norm_eps
            if pre_norm:
                self.norm_pre.eps = norm_eps
        self.head = nn.Linear(embed_dim, num_classes)
        if distilled:
            self.head_dist = nn.Linear(embed_dim, num_classes)
        self._link_views()
        self._cfg = vit_config(img_size, patch_size, in_chans, num_classes, embed_dim, depth, num_heads, mlp_ratio,
                               distilled, self.blocks[0].norm1.eps, self.norm.eps, pre_norm=pre_norm, act=act_layer)
        self._engine = None
        self._weights_version = None
        self.engine_flags = 0
        self._rule_flags = 0                   # ViT_orig_LRP sets TE_FLAG_RULES_LRP (the modules/layers_lrp.py rule library)
        self._init_weights()

    def _link_views(self):
        # a weak back-reference, kept out of the module tree: a strong one would make model <-> view a reference cycle,
        # so a dropped model and its engine's device memory (weights, derived copies, workspace) would live on until
        # Python's cyclic garbage collector happened to run
        for i, blk in enumerate(self.blocks):
            blk.attn._owner = weakref.ref(self)
            blk.attn._layer = i

    def __setstate__(self, state):             # pickle / copy.deepcopy: the views answer for the new model
        super().__setstate__(state)
        self._link_views()

    def _init_weights(self):
        # reference init (ViT_LRP.py:276-299): trunc_normal(.02) for Linear / pos / cls, LayerNorm 1/0
        nn.init.trunc_normal_(self.pos_embed, std=.02)
        nn.init.trunc_normal_(self.cls_token, std=.02)
        if self.distilled:
            nn.init.trunc_normal_(self.dist_token, std=.02)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.LayerNorm):
                nn.init.constant_(m.bias, 0)
                nn.init.constant_(m.weight, 1.0)

    @property
    def no_weight_decay(self):
        return {'pos_embed', 'cls_token'}

    # ---- engine plumbing --------------------------------------------------------------------------
    def _version(self):
        return tuple(p._version for p in self.parameters()) + (str(self.pos_embed.device),)

    def engine(self):
        """The CUDA engine holding a packed copy of the (frozen) parameters; re-packed when they change."""
        dev = self.pos_embed.device
        if dev.type != "cuda":
            raise RuntimeError("the CUDA engine has no CPU path: move the model to a CUDA device (model.cuda())")
        v = self._version()
        if self._engine is None or self._engine.device != dev:
            self._engine = ViTEngine(self._cfg, device=dev, flags=self.engine_flags | self._rule_flags)
            self._weights_version = None
        if self._weights_version != v:
            self._engine.load_state_dict(self.state_dict())
            self._weights_version = v
        self._engine.flags = self.engine_flags | self._rule_flags
        return self._engine

    def _engine_tensor(self, name, layer):
        if self._engine is None or self._engine.last_batch <= 0:
            raise RuntimeError("no saved activations: call model(x) (and model.relprop(...)) first")
        return self._engine.tensor(name, layer)

    # ---- model(x) -----------------------------------------------------------------------------------
    def forward(self, x):
        H, W = x.shape[-2:]
        assert H == self.patch_embed.img_size[0] and W == self.patch_embed.img_size[1], \
            f"Input image size ({H}*{W}) doesn't match model ({self.patch_embed.img_size[0]}*{self.patch_embed.img_size[1]})."
        return self.engine().forward(x)

    # ---- model.relprop(...) -------------------------------------------------------------------------
    def relprop(self, cam=None, method="transformer_attribution", is_ablation=False, start_layer=0, **kwargs):
        """``ViT_LRP.py:324-398``.  ``cam`` is the one-hot class-relevance seed [B,C] (``generate_LRP`` passes
        the same one-hot it back-propagates, ViT_explanation_generator.py:31-40); the engine derives the class
        index from it and runs gradient + relprop + rollout in one call.  ``alpha`` (default 1) selects the
        LRP-alpha-beta rule, beta = alpha - 1, in every Linear.relprop, for every method that runs the relprop."""
        alpha = kwargs.get("alpha", 1)
        eng = self.engine()
        index = cam.argmax(dim=-1).to(torch.int32) if cam is not None else None
        first = 2 if self.distilled else 1
        if method in ("transformer_attribution", "grad"):
            maps, _ = eng.attribute(index=index, start_layer=start_layer, alpha=alpha)
            return maps
        if method == "full":                                   # :337-343: relevance of every pixel, channels summed
            return eng.relprop_pixels(index=index, alpha=alpha)
        # secondary methods (:345-398): head reductions of the saved per-block tensors
        if method == "rollout":                                # attn_cam of every block -> rollout
            eng.attribute(index=index, start_layer=0, flags=eng.flags | _lib.FLAG_KEEP_ALL_CAMS, alpha=alpha)
            cams = [ops.head_reduce(blk.attn.get_attn_cam(), mode="relu_mean") for blk in self.blocks]
            return compute_rollout_attention(cams, start_layer=start_layer)[:, 0, first:]
        if method in ("last_layer", "second_layer"):
            l = len(self.blocks) - 1 if method == "last_layer" else 1
            eng.attribute(index=index, start_layer=l, alpha=alpha)     # the relprop stops at attn_cam of block l
            attn = self.blocks[l].attn
            c = ops.head_reduce(attn.get_attn_cam(), attn.get_attn_gradients() if is_ablation else None, mode="relu_mean")
            return c[:, 0, first:]
        if method == "last_layer_attn":
            return ops.head_reduce(self.blocks[-1].attn.get_attn(), mode="relu_mean")[:, 0, first:]
        raise ValueError("unknown method %r" % (method,))


def _conv_filter(state_dict, patch_size=16):
    """``ViT_LRP.py:401-408``: manual-patchify linear weights -> conv weights."""
    out = {}
    for k, v in state_dict.items():
        if 'patch_embed.proj.weight' in k:
            v = v.reshape((v.shape[0], 3, patch_size, patch_size))
        out[k] = v
    return out


def _no_pretrained(pretrained):
    if pretrained:
        raise RuntimeError("pretrained weights are not downloadable here; load a state_dict with "
                           "model.load_state_dict(...) (timm key names)")


def vit_base_patch16_224(pretrained=False, **kwargs):
    _no_pretrained(pretrained)
    return VisionTransformer(patch_size=16, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True, **kwargs)


def vit_large_patch16_224(pretrained=False, **kwargs):
    _no_pretrained(pretrained)
    return VisionTransformer(patch_size=16, embed_dim=1024, depth=24, num_heads=16, mlp_ratio=4, qkv_bias=True, **kwargs)


def deit_base_patch16_224(pretrained=False, **kwargs):
    _no_pretrained(pretrained)
    return VisionTransformer(patch_size=16, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True, **kwargs)


def deit_base_distilled_patch16_224(pretrained=False, **kwargs):
    _no_pretrained(pretrained)
    return VisionTransformer(patch_size=16, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True,
                             distilled=True, **kwargs)
